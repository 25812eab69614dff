"""Per-GPU iteration plan: the replacement for one `session.run` of the
reference's iteration graph.

The reference builds a TF1 graph per AdaNet iteration
(adanet/core/iteration.py:506-816) and executes every subnetwork's and every
candidate ensemble's train op in one `session.run` per step through hooks
(adanet/core/iteration.py:150-205,961-996).  Here an :class:`IterationPlan`
owns, for the candidates placed on this GPU, all parameters, activations,
gradients and bookkeeping in HBM and enqueues the hand-written sm_90a (H100) kernels
of ``adanet_b200/csrc`` through the C ABI (include/adanet_b200.h).

Dense layers run on the plane-native tensor-core pipeline (csrc/planes.cu): the
minibatch is split into hi/lo planes (fp16 pairs by default, TF32 pairs as the
fallback: csrc/plane_fmt.cuh) once per step and every hidden activation and
back-propagated gradient stays in plane format between GEMMs.  A step is a wave
schedule (IterationPlan._enqueue_waves) of grouped launches built from one op
builder per stage:

  forward layer   -> DenseNet.fwd_op          in adn_dense_fwd_p_group (frozen members too)
  losses, heads   -> CandidatePlan.sub_head_op / EnsembleHead.head_op in adn_head_group
  backward layer  -> CandidatePlan.bwd_op     in adn_dense_bwd_p_group
  optimizers      -> _Optimizer.op            in adn_opt_step_group
  EMA / trace     -> EnsembleHead.book        in adn_head_bookkeeping

With ADN_DENSE_PATH=simt the fp32 CUDA-core ABI is used instead, as an on-device
cross-check: each candidate runs its whole step op by op (adn_dense_fwd /
adn_head_loss / adn_ensemble_head / adn_dense_bwd / adn_opt_step) on its own
stream (CandidatePlan.enqueue_simt_step).

Once shapes are fixed the whole step is captured in a CUDA graph, so a step is
one graph launch.  PyTorch is used for device memory, streams and graphs only.
"""

from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from adanet_b200 import _lib

_HEAD_KIND = {"softmax_xent": _lib.HEAD_SOFTMAX_XENT, "mse": _lib.HEAD_MSE, "sigmoid_xent": _lib.HEAD_SIGMOID_XENT}
_MIX_KIND = {"scalar": _lib.MIX_SCALAR, "vector": _lib.MIX_VECTOR, "matrix": _lib.MIX_MATRIX}
_OPT_KIND = {"sgd": _lib.OPT_SGD, "momentum": _lib.OPT_MOMENTUM, "rmsprop": _lib.OPT_RMSPROP, "adam": _lib.OPT_ADAM,
             "momentum_cosine": _lib.OPT_MOMENTUM_COSINE}
# ("momentum_cosine", lr, momentum, decay_steps[, alpha]): Momentum under tf.train.cosine_decay of the iteration step
_OPT_DEFAULTS = {"sgd": (), "momentum": (), "rmsprop": (0.9, 0.0, 1e-10), "adam": (0.9, 0.999, 1e-8),
                 "momentum_cosine": (0.0,)}
TRACE_FIELDS = ("sub_loss", "ens_loss", "adanet_loss", "ema")
EVAL_METRICS = ("adanet_loss", "loss", "average_loss", "accuracy")


def correct_of(logits: torch.Tensor, labels: torch.Tensor) -> Tuple[int, int]:
  """(correct, total) predictions: arg-max for [B, C>1] logits against int labels, logit > 0 for a single-logit
  (sigmoid) head against {0,1} labels.  Evaluation bookkeeping, not on the step path."""
  if logits.shape[1] > 1:
    return int((logits.argmax(dim=1) == labels.reshape(-1)).sum().item()), int(logits.shape[0])
  return int(((logits.reshape(-1) > 0) == (labels.reshape(-1) > 0.5)).sum().item()), int(logits.numel())


def accuracy_of(logits: torch.Tensor, labels: torch.Tensor) -> float:
  """Fraction of correct predictions (correct_of)."""
  correct, total = correct_of(logits, labels)
  return correct / total


def _check_head_ws(rows: int, logits_dim: int, n_members: int, have: int):
  """A head launched on the first `rows` examples of buffers sized for the static batch must fit the workspace
  allocated for that batch."""
  need = _lib.query(_lib.Q_HEAD_WS, rows, logits_dim, n_members)
  if need > have:
    raise RuntimeError("head workspace of %d bytes is too small for %d rows (needs %d)" % (have, rows, need))


def _load_rows(x_buf: torch.Tensor, labels_buf: Optional[torch.Tensor], x, y) -> int:
  """Copies an evaluation batch of b <= batch examples into the first b rows of the static-batch buffers and zeroes
  the rest; returns b.  `y` may be None (predict): the labels buffer is then left alone."""
  x = torch.as_tensor(x)
  b, batch = int(x.shape[0]), int(x_buf.shape[0])
  if not 0 < b <= batch:
    raise ValueError("an evaluation batch of %d examples does not fit the static batch of %d" % (b, batch))
  x_buf[:b].copy_(x.reshape((b,) + tuple(x_buf.shape[1:])), non_blocking=True)
  x_buf[b:].zero_()
  if y is not None:
    labels_buf[:b].copy_(torch.as_tensor(y).reshape((b,) + tuple(labels_buf.shape[1:])), non_blocking=True)
    labels_buf[b:].zero_()
  return b


def _stream_ptr(stream: Optional[torch.cuda.Stream] = None) -> int:
  s = stream if stream is not None else torch.cuda.current_stream()
  return s.cuda_stream


def _require_cuda():
  if not torch.cuda.is_available():
    raise _lib.AdnError("adanet_b200 engine needs a CUDA device (sm_90a); there is no CPU fallback.")
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  return lib


def planes_enabled() -> bool:
  """True unless the fp32 SIMT cross-check path is forced (adn_set_dense_path / ADN_DENSE_PATH=simt)."""
  return _lib.query(_lib.Q_DENSE_FWD_PATH, 1 << 20, 1024, 1024) == _lib.PATH_TCGEN05


def new_planes(rows: int, cols: int, device) -> torch.Tensor:
  """Zero-initialised split-plane tensor in the CURRENT plane format (include/adanet_b200.h: the K padding must
  stay zero)."""
  return torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, rows, cols) // 4,), dtype=torch.float32, device=device)


def kept_indices(keep_previous, n_frozen: int) -> List[int]:
  """Previous-ensemble members a candidate keeps: True -> all, False -> none, else the given indices (partial pruning
  by a custom Strategy, adanet/core/ensemble_builder.py:367-388)."""
  if keep_previous is True:
    return list(range(n_frozen))
  if keep_previous is False or keep_previous is None:
    return []
  idx = [int(i) for i in keep_previous]
  if any(i < 0 or i >= n_frozen for i in idx) or sorted(set(idx)) != idx:
    raise ValueError("kept previous members must be increasing indices below %d, got %r" % (n_frozen, idx))
  return idx


def gammas(lam: float, beta: float, complexities: Sequence[float]) -> List[float]:
  """gamma_k = lambda * complexity_k + beta of each member (weighted.py:351-358, _compute_adanet_gamma), evaluated in
  fp32 like the graph does."""
  return [float(np.float32(beta) if lam == 0.0 else np.float32(np.float32(lam) * np.float32(c) + np.float32(beta)))
          for c in complexities]


def matrix_member_logits(lib, members, mwp, mw_logits, xp, sp: int, mw=None, mw_l1=None):
  """MATRIX mixture weights (weighted.py:449): weighted_k = last_layer_k @ W_k of every member by the plane GEMM, into
  mw_logits[k]; with `mw`, also ||W_k||_1 into mw_l1[k] for the regulariser, right after member k's GEMM."""
  for k, m in enumerate(members):
    batch, C = mw_logits[k].shape
    _lib.check(lib.adn_dense_fwd_p(m.last_layer_planes(xp).data_ptr(), mwp[k].data_ptr(), None, None,
                                   mw_logits[k].data_ptr(), batch, m.last_layer_dim, C, _lib.ACT_NONE, sp),
               "adn_dense_fwd_p")
    if mw is not None:
      _lib.check(lib.adn_l1_norm(mw[k].data_ptr(), mw[k].numel(), mw_l1.data_ptr() + 4 * k, sp), "adn_l1_norm")


def _select_prev(prev_mixture_weights, idx: List[int]):
  """The warm-start weights of the kept members (SCALAR [N] / VECTOR [N,C] array, or the MATRIX list)."""
  if prev_mixture_weights is None:
    return None
  if isinstance(prev_mixture_weights, list):
    return [prev_mixture_weights[i] for i in idx]
  return np.asarray(prev_mixture_weights)[idx]


class _GradArena:
  """One flat fp32 buffer that hands out 64 B-aligned views: every tensor a row-sharded candidate must average across
  its ranks (weight / bias gradients, mixture-weight gradients, the loss scalars) lives in it, so the cross-rank
  exchange of a step is ONE all-reduce per candidate."""

  def __init__(self, device, capacity: int):
    self.buf = torch.zeros((capacity,), dtype=torch.float32, device=device)
    self.off = 0

  def __call__(self, shape) -> torch.Tensor:
    shape = tuple(int(v) for v in (shape if isinstance(shape, (tuple, list, torch.Size)) else (shape,)))
    n = int(np.prod(shape)) if shape else 1
    if self.off + n > self.buf.numel():
      raise RuntimeError("gradient arena too small")
    t = self.buf[self.off:self.off + n].view(shape)
    self.off += (n + 15) // 16 * 16
    return t

  def used(self) -> torch.Tensor:
    return self.buf[:self.off]


class ShardComm:
  """The ranks that train one row-sharded candidate (distributed/exchange.sharded_placement): shard `index` of `count`.

  `average_(t)` replaces t by its mean over the group, bit-identical on every member: NCCL all-reduce (AVG) on the
  stream of the step -- captured into the step's CUDA graph -- or, when the job runs on gloo (CPU tests, several
  ranks sharing one GPU), through host memory."""

  def __init__(self, ranks: Sequence[int], my_rank: int, group):
    self.ranks = [int(r) for r in ranks]
    self.count = len(self.ranks)
    self.index = self.ranks.index(int(my_rank))
    self.group = group

  @property
  def graph_safe(self) -> bool:
    import torch.distributed as dist
    return dist.get_backend() == "nccl"

  def average_(self, t: torch.Tensor):
    import torch.distributed as dist
    if dist.get_backend() == "nccl":
      dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group)
    else:
      h = t.cpu()
      dist.all_reduce(h, op=dist.ReduceOp.SUM, group=self.group)
      t.copy_(h / float(self.count))      # count is a power of two: exact


def grad_log2_scale(batch: int) -> int:
  """Power-of-two scale of every gradient plane tensor (csrc/plane_fmt.cuh): mean-reduced losses give dlogits of
  O(1/batch), below fp16's normal range; 2^ceil(log2 batch) brings them back to O(1).  TF32 planes need none."""
  return int(math.ceil(math.log2(max(batch, 1)))) if _lib.plane_format() == _lib.PLANES_F16 else 0


@dataclass
class SubnetworkPlanSpec:
  """What a Builder lowers to for the dense hot path.

  name/complexity follow adanet/examples/simple_dnn.py:61-131; `dims` is
  [d0, H, ..., H, logits_dim]; `optimizer` is ("sgd", lr) | ("momentum", lr, m)
  | ("rmsprop", lr[, rho, mu, eps]) | ("adam", lr[, b1, b2, eps]) with TF1
  semantics; `ws`/`bs` are the initial kernels W[in,out] / biases (NumPy fp32).

  A SimpleCNN subnetwork (customizing_adanet.ipynb SimpleCNNBuilder) is the same dense stack behind a conv stem:
  `ws[0]` is then the 4-D HWIO kernel [3,3,Cin,F] and `bs[0]` its bias, `image_shape` = (H, W, Cin) of the NHWC
  minibatch, and `dims[0]` = (H/2)(W/2)F, the flattened pooled feature map the first dense layer consumes.
  """
  name: str
  dims: Sequence[int]
  complexity: float
  optimizer: tuple
  ws: List[np.ndarray]
  bs: List[np.ndarray]
  shared: Optional[dict] = None
  image_shape: Optional[Tuple[int, int, int]] = None
  # bagging (adanet/autoensemble/common.py:151-180): the subnetwork trains on minibatches of its OWN input_fn
  # (before the step's main pass, :43-56) and only its forward on the shared minibatch feeds the ensembles
  own_input: bool = False
  # Subnetwork.last_layer is the logits tensor itself (autoensemble/common.py:115-118) rather than the activation
  # feeding the logits layer; only MATRIX mixture weights read it
  last_layer_is_logits: bool = False
  # tf.layers.dropout after hidden layers in TRAIN mode (simple_dnn.py:80-81): per hidden layer (rate, seed) or None
  dropout: Optional[list] = None


@dataclass
class EnsemblerPlanSpec:
  """ComplexityRegularizedEnsembler arguments (adanet/ensemble/weighted.py:228-251); kind="mean" is the
  MeanEnsembler (adanet/ensemble/mean.py:92-135)."""
  optimizer: Optional[tuple] = None
  mixture_weight_type: str = "scalar"
  adanet_lambda: float = 0.0
  adanet_beta: float = 0.0
  use_bias: bool = False
  name: str = "complexity_regularized"
  legacy_train_op: bool = False
  warm_start_mixture_weights: bool = False   # weighted.py:270-285,487-516
  kind: str = "complexity_regularized"
  # custom `mixture_weight_initializer` (weighted.py:360-366,419-428): fn(num_members, last_layer_dim, logits_dim) ->
  # the initial weight of ONE member (shape [] / [C] / [D_k, C]); None = the reference defaults (1/N, zeros for MATRIX)
  initial_weight_fn: Optional[object] = None


def _opt_hyper(spec: tuple) -> Tuple[int, List[float]]:
  kind = spec[0]
  vals = list(spec[1:])
  defaults = _OPT_DEFAULTS[kind]
  n_fixed = {"sgd": 1, "momentum": 2, "rmsprop": 1, "adam": 1, "momentum_cosine": 3}[kind]
  extra = vals[n_fixed:]
  vals = vals[:n_fixed] + list(extra) + list(defaults[len(extra):])
  return _OPT_KIND[kind], [float(v) for v in vals]


class _Optimizer:
  """Device-resident optimizer state for one group of parameter tensors."""

  def __init__(self, spec: tuple, params: List[torch.Tensor], planes: Optional[List[Optional[torch.Tensor]]] = None):
    self.kind, self.hyper = _opt_hyper(spec)
    self.params = params
    self.planes = planes
    if planes is not None:
      self._planes = _lib.ptr_array([pl.data_ptr() if pl is not None else None for pl in planes])
      self._cols = _lib.i64_array([p.shape[-1] if pl is not None else 0 for p, pl in zip(params, planes)])
    dev = params[0].device
    n_slots = {_lib.OPT_SGD: 0, _lib.OPT_MOMENTUM: 1, _lib.OPT_RMSPROP: 2, _lib.OPT_ADAM: 2,
               _lib.OPT_MOMENTUM_COSINE: 1}[self.kind]
    self.slot0 = [torch.zeros_like(p) for p in params] if n_slots >= 1 else None
    self.slot1 = [torch.zeros_like(p) for p in params] if n_slots >= 2 else None
    if self.kind == _lib.OPT_RMSPROP:
      for s in self.slot0:
        s.fill_(1.0)   # TF RMSProp: ms initialised to ones
    self.step_dev = (torch.zeros((), dtype=torch.int64, device=dev)
                     if self.kind in (_lib.OPT_ADAM, _lib.OPT_MOMENTUM_COSINE) else None)
    self._p = _lib.ptr_array([p.data_ptr() for p in params])
    self._s0 = _lib.ptr_array([s.data_ptr() for s in self.slot0]) if self.slot0 else None
    self._s1 = _lib.ptr_array([s.data_ptr() for s in self.slot1]) if self.slot1 else None
    self._sizes = _lib.i64_array([p.numel() for p in params])
    self._hyper = _lib.f32_array(self.hyper)

  def state(self) -> Dict[str, np.ndarray]:
    out = {}
    for name, slots in (("s0", self.slot0), ("s1", self.slot1)):
      if slots:
        for i, t in enumerate(slots):
          out["%s_%d" % (name, i)] = t.cpu().numpy()
    if self.step_dev is not None:
      out["step"] = self.step_dev.cpu().numpy()
    return out

  def load_state(self, st: Dict[str, np.ndarray]):
    for name, slots in (("s0", self.slot0), ("s1", self.slot1)):
      if slots:
        for i, t in enumerate(slots):
          t.copy_(torch.as_tensor(st["%s_%d" % (name, i)]))
    if self.step_dev is not None:
      self.step_dev.copy_(torch.as_tensor(st["step"]))

  def op(self, grads: List[torch.Tensor]) -> "_lib.OptOp":
    """This optimizer's update as an adn_opt_op (adn_opt_step_group applies several in one launch).  The pointer
    arrays it references are kept alive on `self`."""
    self._g = _lib.ptr_array([t.data_ptr() for t in grads])
    cast = lambda a, ty: ctypes.cast(a, ctypes.POINTER(ty)) if a is not None else None
    return _lib.OptOp(self.kind, len(self.params), cast(self._p, ctypes.c_void_p), cast(self._g, ctypes.c_void_p),
                      cast(self._s0, ctypes.c_void_p), cast(self._s1, ctypes.c_void_p),
                      cast(self._sizes, ctypes.c_int64), cast(self._hyper, ctypes.c_float),
                      self.step_dev.data_ptr() if self.step_dev is not None else None,
                      cast(self._planes, ctypes.c_void_p) if self.planes is not None else None,
                      cast(self._cols, ctypes.c_int64) if self.planes is not None else None)

  def apply(self, lib, grads: List[torch.Tensor], stream_ptr: int):
    """This update alone: a one-op adn_opt_step_group."""
    _lib.check(lib.adn_opt_step_group((_lib.OptOp * 1)(self.op(grads)), 1, stream_ptr), "adn_opt_step_group")


class DenseNet:
  """Parameters + activation buffers of one dense subnetwork on one GPU.

  Forward: h_i = relu(h_{i-1} @ W_i + b_i), logits = h_L @ W_o + b_o
  (adanet/examples/simple_dnn.py:70-86).  Used forward-only for frozen
  members (adanet/core/iteration.py:568-579).
  """

  def __init__(self, name: str, dims: Sequence[int], ws, bs, complexity: float, batch: int,
               device: torch.device, iteration: int = 0, shared: Optional[dict] = None,
               image_shape: Optional[Sequence[int]] = None, dropout: Optional[list] = None):
    """`dropout`: per hidden layer (rate, seed) or None -- applied only by `fwd_op(..., step_dev=...)`, i.e. on the
    TRAIN-mode forward of a candidate; frozen members and evaluation replay without it (iteration.py:568-579)."""
    self.name, self.dims, self.complexity, self.iteration = name, list(dims), float(complexity), iteration
    self.dropout = list(dropout) if dropout else None
    self.shared = shared or {}
    self.batch = batch
    self.device = device
    # conv stem (SimpleCNN): a 4-D HWIO first kernel; conv3x3+ReLU+maxpool+flatten into the planes of dims[0]
    self.stem = None
    self.image_shape = tuple(int(v) for v in image_shape) if image_shape is not None else None
    if len(ws) and np.ndim(ws[0]) == 4:
      if self.image_shape is None:
        raise ValueError("subnetwork %s has a conv stem but no image_shape" % name)
      h, w, cin = self.image_shape
      k = np.ascontiguousarray(ws[0], dtype=np.float32)
      if k.shape[:3] != (3, 3, cin) or dims[0] != (h // 2) * (w // 2) * k.shape[3]:
        raise ValueError("conv stem of %s: kernel %s / image %s do not give dims[0]=%d" % (name, k.shape, self.image_shape, dims[0]))
      if not planes_enabled():
        raise NotImplementedError("conv-stem subnetworks run on the plane path only")
      self.stem = dict(h=h, w=w, cin=cin, f=int(k.shape[3]))
      self.stem_k = torch.as_tensor(k).to(device)
      self.stem_b = torch.as_tensor(np.ascontiguousarray(bs[0], dtype=np.float32)).to(device)
      self.stem_out = new_planes(batch, dims[0], device)
      self.stem_arg = torch.zeros((batch * dims[0] // 16,), dtype=torch.int32, device=device)
      ws, bs = ws[1:], bs[1:]
    self.in_dim = int(np.prod(self.image_shape)) if self.stem else self.dims[0]
    self.fmt = _lib.plane_format()
    assert len(ws) == len(dims) - 1
    self.ws = [torch.as_tensor(np.ascontiguousarray(w, dtype=np.float32)).to(device) for w in ws]
    self.bs = [torch.as_tensor(np.ascontiguousarray(b, dtype=np.float32)).to(device) for b in bs]
    for i, w in enumerate(self.ws):
      if tuple(w.shape) != (dims[i], dims[i + 1]):
        raise ValueError("kernel %d of %s has shape %s, want %s" % (i, name, tuple(w.shape), (dims[i], dims[i + 1])))
    self.planes = planes_enabled()
    n = len(self.ws)
    if self.planes:
      # hidden activations live as split planes; only the logits are dense fp32
      self.acts = [None] * (n - 1) + [torch.empty((batch, dims[-1]), dtype=torch.float32, device=device)]
      self.hp = [new_planes(batch, d, device) for d in dims[1:-1]]
      self.wps = [new_planes(dims[i], dims[i + 1], device) for i in range(n)]
      self.refresh_planes()
      self.fwd_ws_bytes, self.fwd_ws = 0, None
    else:
      self.acts = [torch.empty((batch, d), dtype=torch.float32, device=device) for d in dims[1:]]
      self.hp, self.wps = None, None
      fwd_ws = max(_lib.query(_lib.Q_DENSE_FWD_WS, batch, dims[i], dims[i + 1]) for i in range(n))
      self.fwd_ws_bytes = fwd_ws
      self.fwd_ws = torch.empty((max(fwd_ws, 16),), dtype=torch.uint8, device=device)

  def ensure_format(self):
    """Re-creates the plane buffers when the process-wide plane format changed since this net was built (the
    fp16 -> TF32 fallback after an overflow, core/search.py)."""
    if not self.planes or self.fmt == _lib.plane_format():
      return
    self.fmt = _lib.plane_format()
    n = len(self.ws)
    self.hp = [new_planes(self.batch, d, self.device) for d in self.dims[1:-1]]
    self.wps = [new_planes(self.dims[i], self.dims[i + 1], self.device) for i in range(n)]
    if self.stem:
      self.stem_out = new_planes(self.batch, self.dims[0], self.device)
    self.refresh_planes()

  def refresh_planes(self):
    """Re-splits every kernel into its planes (after the dense weights were written from outside the engine,
    e.g. the end-of-iteration broadcast of the winner)."""
    if not self.planes:
      return
    sp = torch.cuda.current_stream(self.device).cuda_stream
    lib = _lib.load()
    for w, wp in zip(self.ws, self.wps):
      _lib.check(lib.adn_planes_split(w.data_ptr(), w.shape[0], w.shape[1], wp.data_ptr(), sp), "adn_planes_split")

  @property
  def logits(self) -> torch.Tensor:
    return self.acts[-1]

  def last_layer_planes(self, xp: torch.Tensor) -> torch.Tensor:
    """Split planes of the last layer (MATRIX mixture weights multiply it, weighted.py:449): the last hidden
    activation, or the input itself for a linear model (simple_dnn.py:70-78)."""
    return self.hp[-1] if len(self.dims) > 2 else (self.stem_out if self.stem else xp)

  def all_params(self) -> List[torch.Tensor]:
    """Every trainable tensor (what the end-of-iteration broadcast of the winner moves)."""
    return ([self.stem_k, self.stem_b] if self.stem else []) + self.ws + self.bs

  def stem_forward(self, lib, x: torch.Tensor, sp: int):
    """images [batch, H*W*Cin] (NHWC) -> planes of the flattened pooled features + the pool arg-max."""
    st = self.stem
    _lib.check(lib.adn_conv_stem_fwd(x.data_ptr(), self.stem_k.data_ptr(), self.stem_b.data_ptr(), self.stem_out.data_ptr(),
                                     self.stem_arg.data_ptr(), self.batch, st["h"], st["w"], st["cin"], st["f"], sp),
               "adn_conv_stem_fwd")

  @property
  def last_layer_dim(self) -> int:
    return self.dims[-2]

  @property
  def last_layer(self) -> torch.Tensor:
    """Last hidden activation as dense fp32 [batch, d] (merged from its planes on demand)."""
    if len(self.dims) < 3:
      return None
    if not self.planes:
      return self.acts[-2]
    out = torch.empty((self.batch, self.dims[-2]), dtype=torch.float32, device=self.device)
    _lib.check(_lib.load().adn_planes_merge(self.hp[-1].data_ptr(), self.batch, self.dims[-2], out.data_ptr(),
                                            torch.cuda.current_stream(self.device).cuda_stream), "adn_planes_merge")
    return out

  def fwd_op(self, i: int, xp: torch.Tensor, step_dev: Optional[torch.Tensor] = None, row0: int = 0) -> "_lib.FwdOp":
    """Layer i as an adn_fwd_op (plane path): hidden layers write planes, the logits layer dense fp32.  With
    `step_dev` (the plan's device step counter) the forward is the TRAIN-mode one: hidden layers with dropout draw
    their keep mask for that step in the epilogue -- for the rows row0, row0 + 1, ... of the minibatch when this net
    trains a row slice of it."""
    last = i == len(self.ws) - 1
    src = (self.stem_out if self.stem else xp) if i == 0 else self.hp[i - 1]
    op = _lib.FwdOp(src.data_ptr(), self.wps[i].data_ptr(), self.bs[i].data_ptr(),
                    None if last else self.hp[i].data_ptr(), self.acts[i].data_ptr() if last else None,
                    self.dims[i], self.dims[i + 1], _lib.ACT_NONE if last else _lib.ACT_RELU, 0)
    d = self.dropout[i] if (self.dropout and step_dev is not None and not last and i < len(self.dropout)) else None
    if d is not None:
      op.dropout_rate, op.dropout_seed, op.dropout_layer = float(d[0]), int(d[1]) & 0xffffffff, i
      op.dropout_row0, op.dropout_step_dev = row0, step_dev.data_ptr()
    return op

  def dx_mul(self, i: int) -> float:
    """Factor on the gradient w.r.t. hidden activation i (the input of layer i + 1): 1 / (1 - rate) when it was
    dropped out in TRAIN mode, else 1."""
    d = self.dropout[i] if (self.dropout and 0 <= i < len(self.dropout)) else None
    return 1.0 / (1.0 - float(d[0])) if d is not None else 1.0

  def forward(self, lib, x: torch.Tensor, sp: int, xp: Optional[torch.Tensor] = None):
    """x: dense fp32 minibatch; xp: its split planes (required on the plane path)."""
    n = len(self.ws)
    if self.planes:
      if self.stem:
        self.stem_forward(lib, x, sp)
      for i in range(n):
        _lib.check(lib.adn_dense_fwd_p_group((_lib.FwdOp * 1)(self.fwd_op(i, xp)), 1, self.batch, sp),
                   "adn_dense_fwd_p_group")
      return
    h = x
    for i in range(n):
      act = _lib.ACT_RELU if i < n - 1 else _lib.ACT_NONE
      _lib.check(lib.adn_dense_fwd(h.data_ptr(), self.ws[i].data_ptr(), self.bs[i].data_ptr(),
                                   self.acts[i].data_ptr(), self.batch, self.dims[i], self.dims[i + 1], act,
                                   self.fwd_ws.data_ptr(), self.fwd_ws_bytes, sp),
                 "adn_dense_fwd")
      h = self.acts[i]

  def numpy_params(self):
    """(kernels, biases) in layer order; a conv stem's HWIO kernel / bias come first."""
    ws, bs = [w.cpu().numpy() for w in self.ws], [b.cpu().numpy() for b in self.bs]
    if self.stem:
      ws, bs = [self.stem_k.cpu().numpy()] + ws, [self.stem_b.cpu().numpy()] + bs
    return ws, bs


class EnsembleHead:
  """One candidate ensemble: mixture weights (+bias) over a list of member subnetworks, its fused head kernel,
  the zero-debiased EMA of its adanet loss and its loss trace (SURVEY.md section 3.3 steps 6-13).

  `member_nets` = kept previous members first, then the candidate's new subnetworks
  (adanet/ensemble/weighted.py:253-300).  The head only reads the members' logits / last layers, so any number
  of heads can share the subnetworks of an iteration (GrowStrategy: one head per new subnetwork; SoloStrategy:
  the new subnetwork alone; AllStrategy: every new subnetwork; adanet/ensemble/strategy.py:79-117).
  """

  def __init__(self, lib, name: str, member_nets: Sequence[DenseNet], n_prev: int, ens: EnsemblerPlanSpec, batch: int,
               logits_dim: int, head: str, decay: float, trace_capacity: int, device: torch.device,
               prev_mixture_weights=None, prev_bias=None, sub_loss: Optional[torch.Tensor] = None, alloc=None,
               row0: int = 0):
    """`alloc(shape)`: where the tensors that a row-sharded candidate averages across ranks are placed (its
    _GradArena); `row0`: first minibatch row of this head when `batch` is a row slice -- members built for the full
    minibatch (frozen ones) are then read from that row on."""
    self.lib, self.name, self.ens = lib, name, ens
    self.batch, self.C, self.head = batch, logits_dim, _HEAD_KIND[head]
    self.member_nets = list(member_nets)
    self.n_prev = n_prev
    n_members = len(self.member_nets)
    f32 = dict(dtype=torch.float32, device=device)
    self.device = device
    self.planes = planes_enabled()
    self.dz_log2 = grad_log2_scale(batch)
    self.kind = getattr(ens, "kind", "complexity_regularized")
    self.mix = _MIX_KIND[ens.mixture_weight_type]
    if self.mix == _lib.MIX_MATRIX:
      # W_k [D_k, C] (zeros, weighted.py:424-428) applied to each member's last layer by the plane GEMM; the
      # head kernel then sees pre-multiplied members and the L1 norms (include/adanet_b200.h)
      if not self.planes:
        raise NotImplementedError("MATRIX mixture weights run on the plane path only (ADN_DENSE_PATH=simt is a cross-check)")
      self.mw = [torch.zeros((m.last_layer_dim, logits_dim), **f32) for m in self.member_nets]
      self.mwp = [new_planes(m.last_layer_dim, logits_dim, device) for m in self.member_nets]
      self.d_mw = [torch.zeros_like(w) for w in self.mw]
      self.mw_logits = [torch.empty((batch, logits_dim), **f32) for _ in self.member_nets]
      self.mw_l1 = torch.zeros((n_members,), **f32)
      self.dens = torch.empty((batch, logits_dim), **f32)
      self.densp = new_planes(batch, logits_dim, device)
      self.mw_ws_bytes = max(_lib.query(_lib.Q_DENSE_BWD_P_WS, batch, m.last_layer_dim, logits_dim) for m in self.member_nets)
      self.mw_ws = torch.empty((self.mw_ws_bytes,), dtype=torch.uint8, device=device)
      self.mix_w = self.mw_l1
    else:
      wshape = (n_members,) if self.mix == _lib.MIX_SCALAR else (n_members, logits_dim)
      self.mix_w = torch.full(wshape, 1.0 / n_members, **f32)
    if getattr(ens, "initial_weight_fn", None) is not None and self.kind != "mean":
      sp0 = torch.cuda.current_stream(device).cuda_stream
      for k, m in enumerate(self.member_nets):
        w0 = np.asarray(ens.initial_weight_fn(n_members, m.last_layer_dim, logits_dim), dtype=np.float32)
        if self.mix == _lib.MIX_MATRIX:
          self.mw[k].copy_(torch.as_tensor(np.ascontiguousarray(w0.reshape(self.mw[k].shape))))
          _lib.check(lib.adn_planes_split(self.mw[k].data_ptr(), self.mw[k].shape[0], self.mw[k].shape[1],
                                          self.mwp[k].data_ptr(), sp0), "adn_planes_split")
        else:
          self.mix_w[k] = torch.as_tensor(np.ascontiguousarray(w0.reshape(tuple(self.mix_w.shape[1:])))).to(device)
    self.bias = torch.zeros((logits_dim,), **f32)
    if self.kind == "mean":
      # MeanEnsembler (adanet/ensemble/mean.py:92-135): the mean of the NEW subnetworks' logits, previous members
      # ignored, nothing trained, no complexity penalty
      n_new = n_members - n_prev
      self.mix_w.zero_()
      self.mix_w[n_prev:] = 1.0 / n_new
    elif ens.warm_start_mixture_weights and prev_mixture_weights is not None and n_prev > 0:
      # kept members and the bias start from the previous ensemble's trained values (weighted.py:270-285,487-516);
      # new members keep the default initialiser for the grown member count
      if self.mix == _lib.MIX_MATRIX:
        sp0 = torch.cuda.current_stream(device).cuda_stream
        for k in range(n_prev):
          self.mw[k].copy_(torch.as_tensor(np.ascontiguousarray(prev_mixture_weights[k], dtype=np.float32)))
          _lib.check(lib.adn_planes_split(self.mw[k].data_ptr(), self.mw[k].shape[0], self.mw[k].shape[1],
                                          self.mwp[k].data_ptr(), sp0), "adn_planes_split")
      else:
        prev = torch.as_tensor(np.ascontiguousarray(prev_mixture_weights, dtype=np.float32)).to(device)
        self.mix_w[:n_prev] = prev.reshape((n_prev,) + tuple(self.mix_w.shape[1:]))
      if prev_bias is not None:
        self.bias.copy_(torch.as_tensor(np.ascontiguousarray(prev_bias, dtype=np.float32)).reshape(logits_dim))
    alloc = alloc if alloc is not None else (lambda shape: torch.zeros(shape, **f32))
    self.d_mix_w = alloc(tuple(self.mix_w.shape))
    self.d_bias = alloc((logits_dim,))
    self.complexities = [m.complexity for m in self.member_nets]
    lam, beta = float(ens.adanet_lambda), float(ens.adanet_beta)
    if self.kind == "mean":
      lam = beta = 0.0
    self.reg_is_zero = int(lam == 0.0 and beta == 0.0)
    self.gammas = gammas(lam, beta, self.complexities)
    self.reg_multiplier = 1.0 if ens.legacy_train_op else 2.0   # SURVEY.md section 3.3 step 11
    self.out3 = alloc((3,))
    self.ens_opt = None
    if ens.optimizer is not None and self.kind != "mean":
      if self.mix == _lib.MIX_MATRIX:
        ens_params = list(self.mw) + ([self.bias] if ens.use_bias else [])
        self._ens_grads = list(self.d_mw) + ([self.d_bias] if ens.use_bias else [])
        self.ens_opt = _Optimizer(ens.optimizer, ens_params, list(self.mwp) + ([None] if ens.use_bias else []))
      else:
        ens_params = [self.mix_w] + ([self.bias] if ens.use_bias else [])
        self._ens_grads = [self.d_mix_w] + ([self.d_bias] if ens.use_bias else [])
        self.ens_opt = _Optimizer(ens.optimizer, ens_params)
    self.ema_state = torch.zeros((3,), **f32)   # {biased, n, value}; candidate.py:101-129
    self.decay = float(decay)
    self.trace = torch.zeros((trace_capacity, 4), **f32)
    self.trace_capacity = trace_capacity
    self.head_ws_bytes = _lib.query(_lib.Q_HEAD_WS, batch, logits_dim, n_members)
    self.head_ws = torch.empty((self.head_ws_bytes,), dtype=torch.uint8, device=device)
    if self.mix == _lib.MIX_MATRIX:
      self._members = _lib.ptr_array([t.data_ptr() for t in self.mw_logits])
    else:
      self._members = _lib.ptr_array([m.logits.data_ptr() + (row0 * logits_dim * 4 if m.batch != batch else 0)
                                      for m in self.member_nets])
    if row0 and self.mix == _lib.MIX_MATRIX:
      raise NotImplementedError("MATRIX mixture weights on a row-sharded candidate")
    self.row0 = row0
    self._gammas = _lib.f32_array(self.gammas)
    # trace row = (sub_loss of the candidate's subnetwork | NaN for a head that owns none, ens_loss, adanet_loss, ema)
    self._nan = torch.full((1,), float("nan"), **f32)
    src0 = sub_loss if sub_loss is not None else self._nan
    self._sub_loss_src = src0
    self._trace_src = _lib.ptr_array([src0.data_ptr(), self.out3.data_ptr(), self.out3.data_ptr() + 8,
                                      self.ema_state.data_ptr() + 8])

  @property
  def groupable(self) -> bool:
    """SCALAR / VECTOR heads run in the grouped launch of the step (adn_head_group); MATRIX heads need their own
    plane GEMMs around the head kernel."""
    return self.mix != _lib.MIX_MATRIX

  def head_op(self, labels, labels_f) -> "_lib.HeadOp":
    """This head as an adn_head_op: ensemble logits, loss, penalty, mixture-weight / bias gradients (steps 6-11)."""
    train_ens = self.ens_opt is not None
    return _lib.HeadOp(self.head, self.mix, ctypes.cast(self._members, ctypes.POINTER(ctypes.c_void_p)),
                       len(self.member_nets), self.reg_is_zero, self.mix_w.data_ptr(), self.bias.data_ptr(),
                       ctypes.cast(self._gammas, ctypes.POINTER(ctypes.c_float)), self.reg_multiplier, 0,
                       labels.data_ptr() + self.row0 * 8 if labels is not None else None,
                       labels_f.data_ptr() + self.row0 * self.C * 4 if labels_f is not None else None, self.out3.data_ptr(),
                       self.d_mix_w.data_ptr() if train_ens else None,
                       self.d_bias.data_ptr() if (train_ens and self.ens.use_bias) else None, None, None, None, 0, 0,
                       self.head_ws.data_ptr(), self.head_ws_bytes)

  def book(self) -> "_lib.HeadBook":
    """EMA + trace row of this head (steps 12-13) as an adn_head_book."""
    return _lib.HeadBook(self.ema_state.data_ptr(), self.out3.data_ptr(), self._sub_loss_src.data_ptr(), self.trace.data_ptr(),
                         self.decay, self.trace_capacity)

  def enqueue_matrix(self, labels, labels_f, sp: int, xp: torch.Tensor):
    """steps 6-11 of a MATRIX head in the wave schedule, on pre-update values: the members' plane GEMMs and L1 norms,
    ensemble logits, loss, penalty and the mixture-weight gradients.  Its EMA, trace row and update run in the
    step's grouped launches."""
    lib, B, C = self.lib, self.batch, self.C
    train_ens = self.ens_opt is not None
    matrix_member_logits(lib, self.member_nets, self.mwp, self.mw_logits, xp, sp, self.mw, self.mw_l1)
    _lib.check(lib.adn_ensemble_head(
        self.head, self.mix, self._members, len(self.member_nets), self.mix_w.data_ptr(), self.bias.data_ptr(),
        self._gammas, self.reg_is_zero, self.reg_multiplier, labels.data_ptr() if labels is not None else None,
        labels_f.data_ptr() if labels_f is not None else None, self.out3.data_ptr(), None,
        self.d_bias.data_ptr() if (train_ens and self.ens.use_bias) else None,
        self.dens.data_ptr() if train_ens else None, None, B, C, self.head_ws.data_ptr(), self.head_ws_bytes, sp),
               "adn_ensemble_head")
    if not train_ens:
      return
    # dW_k = last_layer_k^T @ dLoss/d(ens)  + reg_multiplier * gamma_k * sign(W_k)   (weighted.py:606-617); each dW
    # GEMM is launched alone: its split-K count, and so its bytes, depend on the group it runs in
    _lib.check(lib.adn_planes_split_scaled(self.dens.data_ptr(), B, C, self.densp.data_ptr(), self.dz_log2, sp),
               "adn_planes_split_scaled")
    for k, m in enumerate(self.member_nets):
      op = _lib.BwdOp(m.last_layer_planes(xp).data_ptr(), None, self.densp.data_ptr(), None, None, None,
                      self.d_mw[k].data_ptr(), m.last_layer_dim, C, 0, self.dz_log2, self.mw_ws.data_ptr(),
                      self.mw_ws_bytes, 0.0, 0.0)
      _lib.check(lib.adn_dense_bwd_p_group((_lib.BwdOp * 1)(op), 1, B, sp), "adn_dense_bwd_p_group")
      if not self.reg_is_zero:
        _lib.check(lib.adn_l1_grad_add(self.d_mw[k].data_ptr(), self.mw[k].data_ptr(), self.mw[k].numel(),
                                       self.reg_multiplier * self.gammas[k], sp), "adn_l1_grad_add")

  def enqueue_simt(self, labels, labels_f, step_dev, sp: int):
    """steps 6-13 of a SCALAR / VECTOR head on the SIMT cross-check path, on pre-update values: ensemble logits, loss,
    penalty, mixture-weight gradient, EMA, trace row and mixture-weight update, op by op."""
    lib = self.lib
    train_ens = self.ens_opt is not None
    _lib.check(lib.adn_ensemble_head(
        self.head, self.mix, self._members, len(self.member_nets), self.mix_w.data_ptr(), self.bias.data_ptr(),
        self._gammas, self.reg_is_zero, self.reg_multiplier, labels.data_ptr() if labels is not None else None,
        labels_f.data_ptr() if labels_f is not None else None, self.out3.data_ptr(),
        self.d_mix_w.data_ptr() if train_ens else None,
        self.d_bias.data_ptr() if (train_ens and self.ens.use_bias) else None, None, None, self.batch, self.C,
        self.head_ws.data_ptr(), self.head_ws_bytes, sp), "adn_ensemble_head")
    _lib.check(lib.adn_ema_update(self.ema_state.data_ptr(), self.out3.data_ptr() + 8, self.decay, sp),
               "adn_ema_update")
    _lib.check(lib.adn_record_scalars(self._trace_src, 4, self.trace.data_ptr(), 4, step_dev.data_ptr(),
                                      self.trace_capacity, sp), "adn_record_scalars")
    if train_ens:
      self.ens_opt.apply(lib, self._ens_grads, sp)

  def enqueue_eval(self, labels, labels_f, ens_out: Optional[torch.Tensor], sp: int, xp: Optional[torch.Tensor] = None,
                   rows: Optional[int] = None):
    """Forward-only ensemble logits / loss over the members' current logits (Evaluator, evaluate, predict), on the
    first `rows` examples (default: the whole batch) -- row-major logits make them a prefix of every member's."""
    rows = self.batch if rows is None else rows
    _check_head_ws(rows, self.C, len(self.member_nets), self.head_ws_bytes)
    if self.mix == _lib.MIX_MATRIX:
      matrix_member_logits(self.lib, self.member_nets, self.mwp, self.mw_logits, xp, sp, self.mw, self.mw_l1)
    _lib.check(self.lib.adn_ensemble_head(
        self.head, self.mix, self._members, len(self.member_nets), self.mix_w.data_ptr(), self.bias.data_ptr(),
        self._gammas, self.reg_is_zero, self.reg_multiplier,
        labels.data_ptr() if labels is not None else None, labels_f.data_ptr() if labels_f is not None else None,
        self.out3.data_ptr(), None, None, None, ens_out.data_ptr() if ens_out is not None else None, rows,
        self.C, self.head_ws.data_ptr(), self.head_ws_bytes, sp), "adn_ensemble_head")

  def mixture_weight_tensors(self) -> List[torch.Tensor]:
    """The trained mixture weights as tensors: [w] (SCALAR [N] / VECTOR [N,C]) or the N matrices (MATRIX)."""
    return list(self.mw) if self.mix == _lib.MIX_MATRIX else [self.mix_w]

  def state_dict(self) -> Dict[str, np.ndarray]:
    out = {}
    for i, t in enumerate(self.mixture_weight_tensors()):
      out["mix%d" % i] = t.cpu().numpy()
    out["bias"] = self.bias.cpu().numpy()
    if self.ens_opt is not None:
      for k, v in self.ens_opt.state().items():
        out["ens_opt_" + k] = v
    out["ema_state"] = self.ema_state.cpu().numpy()
    out["trace"] = self.trace.cpu().numpy()
    return out

  def load_state_dict(self, st: Dict[str, np.ndarray]):
    for i, t in enumerate(self.mixture_weight_tensors()):
      t.copy_(torch.as_tensor(st["mix%d" % i]))
    if self.mix == _lib.MIX_MATRIX:
      sp = torch.cuda.current_stream(self.device).cuda_stream
      for w, wp in zip(self.mw, self.mwp):
        _lib.check(self.lib.adn_planes_split(w.data_ptr(), w.shape[0], w.shape[1], wp.data_ptr(), sp), "adn_planes_split")
    self.bias.copy_(torch.as_tensor(st["bias"]))
    if self.ens_opt is not None:
      self.ens_opt.load_state({k[len("ens_opt_"):]: v for k, v in st.items() if k.startswith("ens_opt_")})
    self.ema_state.copy_(torch.as_tensor(st["ema_state"]))
    self.trace.copy_(torch.as_tensor(st["trace"]))


class CandidatePlan:
  """One `*_grow` candidate: its new subnetwork + its ensemble head + EMA.

  Colocating the candidate ensemble with its new subnetwork is possible because
  under GrowStrategy each candidate contains exactly one new subnetwork
  (adanet/ensemble/strategy.py:97-106); SURVEY.md section 8e.
  """

  def __init__(self, lib, spec: SubnetworkPlanSpec, frozen: Sequence[DenseNet], ens: EnsemblerPlanSpec,
               iteration: int, batch: int, logits_dim: int, head: str, decay: float, trace_capacity: int,
               device: torch.device, index: int, prev_mixture_weights=None, prev_bias=None,
               comm: Optional[ShardComm] = None, full_batch: Optional[int] = None):
    """`comm`: this candidate is row-sharded -- `batch` is then the local slice (full_batch / comm.count rows starting
    at row comm.index * batch) and every gradient / loss tensor lives in one arena averaged over comm's ranks."""
    self.lib, self.spec, self.ens, self.index = lib, spec, ens, index
    self.batch, self.C, self.head = batch, logits_dim, _HEAD_KIND[head]
    self.comm = comm
    self.row0 = comm.index * batch if comm is not None else 0
    self.full_batch = full_batch if full_batch is not None else batch
    if comm is not None:
      if getattr(spec, "own_input", False):
        raise NotImplementedError("a bagged subnetwork cannot be row-sharded")
      n_par = sum(int(np.prod(np.shape(w))) + int(np.prod(np.shape(b))) for w, b in zip(spec.ws, spec.bs))
      self.arena = _GradArena(device, n_par + 32 * (2 * len(spec.ws) + 8) + (len(frozen) + 1) * (logits_dim + 1) + 64)
      galloc = self.arena
    else:
      self.arena = None
      galloc = lambda shape: torch.empty(tuple(shape), dtype=torch.float32, device=device)
    self.name = "t{}_{}_grow_{}".format(iteration, spec.name, ens.name)   # iteration.py:633,691-693
    if ens.mixture_weight_type == "matrix" and getattr(spec, "last_layer_is_logits", False):
      # the reference would train W_k [C, C] on the logits (weighted.py:424-453 with common.py:115-118); the engine's
      # MATRIX path multiplies the penultimate activation, which would be a different model: refuse instead
      raise NotImplementedError("MATRIX mixture weights over a subnetwork whose last_layer is its logits (%s) are not "
                                "implemented by the B200 engine; pass last_layer_fn or use SCALAR / VECTOR" % spec.name)
    self.net = DenseNet(spec.name, spec.dims, spec.ws, spec.bs, spec.complexity, batch, device, iteration,
                        spec.shared, spec.image_shape, dropout=getattr(spec, "dropout", None))
    if self.net.dropout and not self.net.planes:
      raise NotImplementedError("dropout runs on the plane path only")
    self.frozen = list(frozen)
    dims = self.net.dims
    f32 = dict(dtype=torch.float32, device=device)
    # gradients and backward scratch
    self.dws = [galloc(w.shape) for w in self.net.ws]
    self.dbs = [galloc(b.shape) for b in self.net.bs]
    self.dlogits = torch.empty((batch, dims[-1]), **f32)
    hid = max(dims[1:-1]) if len(dims) > 2 else 0
    self.planes = self.net.planes
    self.dz_log2 = grad_log2_scale(batch)
    if self.planes:
      # back-propagated gradients as split planes: dlogits + two ping-pong buffers for the hidden layers
      self.dzp_out = new_planes(batch, dims[-1], device)
      self.dzp = [new_planes(batch, hid, device) for _ in range(2)] if hid else []
      self.dz = []
      bwd_ws = max(_lib.query(_lib.Q_DENSE_BWD_P_WS, batch, dims[i], dims[i + 1]) for i in range(len(dims) - 1))
      self.bwd_ws_bytes = max(bwd_ws, _lib.query(_lib.Q_COLSUM_WS, batch, dims[-1]))
      self.bwd_ws = torch.empty((self.bwd_ws_bytes,), dtype=torch.uint8, device=device)
      ws_bytes = 0                    # `workspace` serves the subnetwork's own head op alone
    else:
      self.dz = [torch.empty((batch, hid), **f32) for _ in range(2)] if hid else []
      # `workspace` serves the backward and the subnetwork's own head loss, one after the other on its stream
      ws_bytes = max(_lib.query(_lib.Q_DENSE_BWD_WS, batch, dims[i], dims[i + 1]) for i in range(len(dims) - 1))
    ws_bytes = max(ws_bytes, _lib.query(_lib.Q_HEAD_WS, batch, logits_dim, 1))
    self.workspace = torch.empty((ws_bytes,), dtype=torch.uint8, device=device)
    self.ws_bytes = ws_bytes
    self.sub_out3 = galloc((3,)).zero_()           # {loss, -, -} of the subnetwork's own head
    self.sub_loss = self.sub_out3[:1]
    self._logits_ptr = _lib.ptr_array([self.net.logits.data_ptr()])
    self.bagged = bool(getattr(spec, "own_input", False))
    if self.bagged:
      if not self.planes:
        raise NotImplementedError("bagged subnetworks (own train_input_fn) run on the plane path only")
      self.x_own = torch.empty((batch, self.net.in_dim), **f32)
      self.xp_own = None if self.net.stem else new_planes(batch, self.net.in_dim, device)
      self.labels_own = (torch.empty((batch,), dtype=torch.int64, device=device) if head == "softmax_xent"
                         else torch.empty((batch, logits_dim), **f32))
      self.own_out3 = torch.zeros((3,), **f32)    # {loss, -, -} on the bagged minibatch (not reported by the reference)
      self.own_loss = self.own_out3[:1]
    params, self._grads, planes = [], [], []
    if self.net.stem:
      # conv stem: dense gradient of the pooled features (first dense layer's dX), kernel / bias gradients
      st = self.net.stem
      self.dpool = torch.empty((batch, dims[0]), **f32)
      self.d_stem_k, self.d_stem_b = galloc(self.net.stem_k.shape), galloc(self.net.stem_b.shape)
      self.stem_ws_bytes = _lib.query(_lib.Q_CONV_STEM_BWD_WS, batch, st["cin"], st["f"])
      self.stem_ws = torch.empty((self.stem_ws_bytes,), dtype=torch.uint8, device=device)
      params += [self.net.stem_k, self.net.stem_b]
      self._grads += [self.d_stem_k, self.d_stem_b]
      planes += [None, None]
    for i, (w, b, dw, db) in enumerate(zip(self.net.ws, self.net.bs, self.dws, self.dbs)):
      params += [w, b]
      self._grads += [dw, db]
      planes += [self.net.wps[i] if self.planes else None, None]
    self.sub_opt = _Optimizer(spec.optimizer, params, planes if self.planes else None)
    # the candidate's ensemble: kept previous members + this new subnetwork
    self.ehead = EnsembleHead(lib, self.name, list(frozen) + [self.net], len(frozen), ens, batch, logits_dim, head, decay,
                              trace_capacity, device, prev_mixture_weights=prev_mixture_weights, prev_bias=prev_bias,
                              sub_loss=self.sub_loss, alloc=self.arena, row0=self.row0)
    # the minibatch rows of a row-sharded candidate as its own plane tensor (split from the plan's x every step)
    self.xp_local = new_planes(batch, self.net.in_dim, device) if (comm is not None and not self.net.stem and self.planes) else None
    self.has_head = True      # False when no strategy asked for this subnetwork's `_grow` ensemble

  # the head's state under the names the search / tests use
  mix = property(lambda self: self.ehead.mix)
  mix_w = property(lambda self: self.ehead.mix_w)
  bias = property(lambda self: self.ehead.bias)
  out3 = property(lambda self: self.ehead.out3)
  ema_state = property(lambda self: self.ehead.ema_state)
  trace = property(lambda self: self.ehead.trace)
  trace_capacity = property(lambda self: self.ehead.trace_capacity)
  ens_opt = property(lambda self: self.ehead.ens_opt)

  def enqueue_simt_step(self, x: torch.Tensor, labels: torch.Tensor, labels_f: Optional[torch.Tensor],
                        step_dev: torch.Tensor, sp: int):
    """SURVEY.md section 3.3 steps 1-13 for this candidate on the fp32 SIMT cross-check path, op by op on stream `sp`
    (frozen logits already computed).  The plane path trains on the wave schedule (IterationPlan._enqueue_waves)."""
    lib, net, B, C = self.lib, self.net, self.batch, self.C
    lab = labels.data_ptr() if labels is not None else None
    labf = labels_f.data_ptr() if labels_f is not None else None
    wsp = self.workspace.data_ptr()
    # steps 1-2: subnetwork forward
    net.forward(lib, x, sp)
    # step 3: subnetwork loss + dlogits
    _lib.check(lib.adn_head_loss(self.head, net.logits.data_ptr(), lab, labf, self.sub_loss.data_ptr(),
                                 self.dlogits.data_ptr(), B, C, wsp, self.ws_bytes, sp), "adn_head_loss")
    # steps 6-13: ensemble head on pre-update values, EMA, trace, mixture-weight update
    if self.has_head:
      self.ehead.enqueue_simt(labels, labels_f, step_dev, sp)
    # step 4: backward through the subnetwork's own variables only
    dz = self.dlogits
    for i in range(len(net.ws) - 1, -1, -1):
      xin = x if i == 0 else net.acts[i - 1]
      # dz ping-pong buffers are sized for the widest hidden layer; carve a contiguous [B, d_i] view
      dx = self.dz[i % 2].view(-1)[:B * net.dims[i]].view(B, net.dims[i]) if i > 0 else None
      _lib.check(lib.adn_dense_bwd(xin.data_ptr(), net.ws[i].data_ptr(), dz.data_ptr(),
                                   dx.data_ptr() if dx is not None else None, self.dws[i].data_ptr(),
                                   self.dbs[i].data_ptr(), B, net.dims[i], net.dims[i + 1], 1 if i > 0 else 0,
                                   wsp, self.ws_bytes, sp), "adn_dense_bwd")
      dz = dx
    # steps 4-5 (apply)
    self.sub_opt.apply(lib, self._grads, sp)

  def state_dict(self) -> Dict[str, np.ndarray]:
    """Everything that changes while the candidate trains (the reference persists the same through the TF
    checkpoint: variables, optimizer slots, EMA, per-spec step counters; iteration.py:40-118,172-183)."""
    out = {}
    for i, (w, b) in enumerate(zip(self.net.ws, self.net.bs)):
      out["w%d" % i], out["b%d" % i] = w.cpu().numpy(), b.cpu().numpy()
    if self.net.stem:
      out["stem_k"], out["stem_b"] = self.net.stem_k.cpu().numpy(), self.net.stem_b.cpu().numpy()
    for k, v in self.sub_opt.state().items():
      out["sub_opt_" + k] = v
    out.update(self.ehead.state_dict())
    return out

  def load_state_dict(self, st: Dict[str, np.ndarray]):
    for i, (w, b) in enumerate(zip(self.net.ws, self.net.bs)):
      w.copy_(torch.as_tensor(st["w%d" % i]))
      b.copy_(torch.as_tensor(st["b%d" % i]))
    if self.net.stem:
      self.net.stem_k.copy_(torch.as_tensor(st["stem_k"]))
      self.net.stem_b.copy_(torch.as_tensor(st["stem_b"]))
    self.net.refresh_planes()
    self.sub_opt.load_state({k[len("sub_opt_"):]: v for k, v in st.items() if k.startswith("sub_opt_")})
    self.ehead.load_state_dict(st)

  def mixture_weight_tensors(self) -> List[torch.Tensor]:
    return self.ehead.mixture_weight_tensors()

  # ---- plane path, wave-synchronous schedule (IterationPlan._enqueue_waves) ----
  def load_own_batch(self, x, y):
    """The bagged subnetwork's own minibatch for the next step (its `train_input_fn`, common.py:151-160)."""
    self.x_own.copy_(torch.as_tensor(x).reshape(self.x_own.shape), non_blocking=True)
    self.labels_own.copy_(torch.as_tensor(y).reshape(self.labels_own.shape), non_blocking=True)

  def sub_head_op(self, labels, labels_f, out3: torch.Tensor) -> "_lib.HeadOp":
    """step 3 as an adn_head_op (colsum_only): subnetwork loss into out3[0], dlogits (dense + scaled planes), db of the
    logits layer."""
    return _lib.HeadOp(self.head, _lib.MIX_SCALAR, ctypes.cast(self._logits_ptr, ctypes.POINTER(ctypes.c_void_p)), 1, 1,
                       None, None, None, 1.0, self.dz_log2, labels.data_ptr() + self.row0 * 8 if labels is not None else None,
                       labels_f.data_ptr() + self.row0 * self.C * 4 if labels_f is not None else None,
                       out3.data_ptr(), None,
                       self.dbs[len(self.net.ws) - 1].data_ptr(), self.dlogits.data_ptr(), None, self.dzp_out.data_ptr(),
                       1, 0, self.workspace.data_ptr(), self.ws_bytes)

  def bwd_op(self, k: int, xp: torch.Tensor) -> "_lib.BwdOp":
    """k-th backward wave = layer n-1-k: dW_i, planes of dZ_{i-1} (ReLU mask = sign bits of h_{i-1}) and
    db_{i-1} = colsum(dZ_{i-1})."""
    net, n = self.net, len(self.net.ws)
    i = n - 1 - k
    xin = (net.stem_out if net.stem else xp) if i == 0 else net.hp[i - 1]
    dzp = self.dzp_out if k == 0 else self.dzp[(i + 1) % 2]
    dxp = self.dzp[i % 2] if i > 0 else None
    ws = self.bwd_ws            # waves are serialised on the main stream
    # below a conv stem the first dense layer also produces dX: dense fp32, masked by the sign bits of the pooled
    # features (= ReLU and max-pool routing mask), which is what adn_conv_stem_bwd consumes
    dx = self.dpool if (i == 0 and net.stem) else None
    # hidden activation i - 1 (the input of this layer) may have been dropped out: its sign bits already carry the keep
    # mask, the 1 / (1 - rate) factor rides on dx
    return _lib.BwdOp(xin.data_ptr(), net.wps[i].data_ptr(), dzp.data_ptr(),
                      dxp.data_ptr() if dxp is not None else None, dx.data_ptr() if dx is not None else None,
                      self.dbs[i - 1].data_ptr() if i > 0 else None, self.dws[i].data_ptr(), net.dims[i],
                      net.dims[i + 1], 1 if (i > 0 or dx is not None) else 0, self.dz_log2, ws.data_ptr(),
                      self.bwd_ws_bytes, net.dx_mul(i - 1) if i > 0 else 0.0, 0.0)

  def enqueue_stem_bwd(self, x: torch.Tensor, sp: int):
    """Kernel / bias gradients of the conv stem from the pooled-feature gradient the last backward wave left."""
    st = self.net.stem
    _lib.check(self.lib.adn_conv_stem_bwd(x.data_ptr(), self.net.stem_arg.data_ptr(), self.dpool.data_ptr(),
                                          self.d_stem_k.data_ptr(), self.d_stem_b.data_ptr(), self.batch, st["h"], st["w"],
                                          st["cin"], st["f"], self.stem_ws.data_ptr(), self.stem_ws_bytes, sp),
               "adn_conv_stem_bwd")


class IterationPlan:
  """All work of one AdaNet iteration placed on this GPU."""

  def __init__(self, iteration: int, specs: Sequence[SubnetworkPlanSpec], frozen: Sequence[DenseNet],
               ens: EnsemblerPlanSpec, batch: int, in_dim: int, logits_dim: int, head: str = "softmax_xent",
               adanet_loss_decay: float = 0.9, trace_capacity: int = 4096, device: Optional[torch.device] = None,
               candidate_indices: Optional[Sequence[int]] = None, use_cuda_graph: bool = True,
               multi_stream: bool = True, prev_mixture_weights=None, prev_bias=None,
               ensemble_candidates: Optional[Sequence[tuple]] = None, prev_ens_name: Optional[str] = None,
               shards: Optional[Dict[int, ShardComm]] = None):
    """`ensemble_candidates`: the candidate ensembles whose members all live on this GPU, as
    (global_index, name, [global subnetwork indices], keep_previous[, EnsemblerPlanSpec]); None = one `*_grow` ensemble
    per local subnetwork (GrowStrategy) under `ens`.  Several ensembles may share a subnetwork
    (adanet/ensemble/strategy.py:79-117), and several ensemblers may each build one over the same strategy candidate
    (adanet/core/iteration.py:683-693).  `prev_ens_name`: the ensembler that built the previous iteration's winner --
    only its own heads warm-start from `prev_mixture_weights` / `prev_bias`.
    `shards[global candidate index]`: that candidate is row-sharded over the ranks of the ShardComm and this rank trains
    its slice of the minibatch rows (distributed/exchange.sharded_placement)."""
    self.lib = _require_cuda()
    self.device = device or torch.device("cuda", torch.cuda.current_device())
    self.iteration, self.batch, self.in_dim, self.C, self.head = iteration, batch, in_dim, logits_dim, head
    self.frozen = list(frozen)
    self.fmt = _lib.plane_format()
    for f in self.frozen:
      f.ensure_format()
      if f.batch != batch:
        raise ValueError("frozen member %s was built for batch %d, plan uses %d" % (f.name, f.batch, batch))
    idx = list(candidate_indices) if candidate_indices is not None else list(range(len(specs)))
    warm = lambda e: prev_ens_name is None or prev_ens_name == e.name
    shards = shards or {}
    for i in idx:
      if i in shards and not planes_enabled():
        # the SIMT step reads the minibatch from row 0 on and never averages the gradient arena
        raise NotImplementedError("row-sharded candidates run on the plane path only")
      if i in shards and batch % shards[i].count != 0:
        raise ValueError("batch %d is not divisible by the %d row shards of candidate %d" % (batch, shards[i].count, i))
    self.candidates = [CandidatePlan(self.lib, s, self.frozen, ens, iteration,
                                     batch // shards[i].count if i in shards else batch, logits_dim, head,
                                     adanet_loss_decay, trace_capacity, self.device, i,
                                     prev_mixture_weights=prev_mixture_weights if warm(ens) else None,
                                     prev_bias=prev_bias if warm(ens) else None, comm=shards.get(i), full_batch=batch)
                       for i, s in zip(idx, specs)]
    self.sharded = [c for c in self.candidates if c.comm is not None]
    if self.sharded and ensemble_candidates is not None:
      raise NotImplementedError("row-sharded candidates with explicit ensemble candidates (Solo / All / several ensemblers)")
    if self.sharded and not all(c.comm.graph_safe for c in self.sharded):
      use_cuda_graph = False        # host-memory exchange (gloo) cannot be captured
    for n in list(self.frozen) + [c.net for c in self.candidates]:
      if n.in_dim != in_dim:
        raise ValueError("subnetwork %s consumes %d input values per example, the plan feeds %d" % (n.name, n.in_dim, in_dim))
    # candidate ensembles: (global index, head, side-stream slot).  A `*_grow` ensemble over one local subnetwork
    # is that CandidatePlan's own head; anything else (solo, all, ...) gets a head of its own over shared nets.
    by_index = {c.index: k for k, c in enumerate(self.candidates)}
    self.heads: List[tuple] = []
    if ensemble_candidates is None:
      self.heads = [(c.index, c.ehead, k) for k, c in enumerate(self.candidates)]
    else:
      for c in self.candidates:
        c.has_head = False
      for ec in ensemble_candidates:
        gidx, name, builders, keep_prev = ec[:4]
        e = ec[4] if len(ec) > 4 and ec[4] is not None else ens
        local = [by_index[b] for b in builders]        # KeyError = a member lives on another rank (caller's bug)
        full_name = "t{}_{}_{}".format(iteration, name, e.name)              # iteration.py:691-693
        own = self.candidates[local[0]]
        kidx = kept_indices(keep_prev, len(self.frozen))
        keeps_all = len(kidx) == len(self.frozen)
        if (len(local) == 1 and keeps_all and name == "{}_grow".format(own.spec.name) and e is ens and not own.has_head):
          own.has_head = True
          self.heads.append((gidx, own.ehead, local[0]))
          continue
        if not planes_enabled():
          raise NotImplementedError("ensembles that share subnetworks run on the plane path only")
        members = [self.frozen[i] for i in kidx] + [self.candidates[k].net for k in local]
        h = EnsembleHead(self.lib, full_name, members, len(kidx), e, batch, logits_dim,
                         head, adanet_loss_decay, trace_capacity, self.device,
                         prev_mixture_weights=_select_prev(prev_mixture_weights, kidx) if (kidx and warm(e)) else None,
                         prev_bias=prev_bias if (kidx and warm(e)) else None,
                         sub_loss=own.sub_loss if len(local) == 1 else None)
        self.heads.append((gidx, h, local[0]))
    self.x = torch.empty((batch, in_dim), dtype=torch.float32, device=self.device)
    # split planes of the minibatch, produced once per step and shared by every member and candidate
    self.xp = new_planes(batch, in_dim, self.device) if planes_enabled() else None
    self.labels = torch.empty((batch,), dtype=torch.int64, device=self.device) if head == "softmax_xent" else None
    self.labels_f = (torch.empty((batch, logits_dim), dtype=torch.float32, device=self.device)
                     if head != "softmax_xent" else None)
    self.step_dev = torch.zeros((), dtype=torch.int64, device=self.device)
    self.steps_done = 0
    self.trace_capacity = trace_capacity
    self.use_cuda_graph = use_cuda_graph
    self.multi_stream = multi_stream and len(self.candidates) > 1
    # side streams of the SIMT schedule, one per candidate
    self.streams = ([torch.cuda.Stream(device=self.device) for _ in self.candidates]
                    if (self.multi_stream and self.xp is None) else [])
    self._graph = None
    self._warmed = False      # set by the first (eager) step
    self._stage = None
    self.carried_overflow = False     # set by a resume from an in-flight state saved after an fp16 overflow
    self.launches_per_step = None

  # -- staging -------------------------------------------------------------
  def load_batch(self, x, y):
    """Copies one minibatch into the plan's fixed staging buffers (H2D when the
    source is host memory; pinned sources copy asynchronously)."""
    x = torch.as_tensor(x)
    y = torch.as_tensor(y)
    self.x.copy_(x.reshape(self.batch, self.in_dim), non_blocking=True)
    if self.labels is not None:
      self.labels.copy_(y.reshape(self.batch), non_blocking=True)
    else:
      self.labels_f.copy_(y.reshape(self.batch, self.C), non_blocking=True)

  def stage_batch(self, x, y):
    """Starts copying the NEXT minibatch into a second set of device buffers on a copy stream, so the
    host->device transfer of step i+1 runs under the kernels of step i; `train_step()` without arguments then
    consumes it (device-to-device move into the graph's fixed input buffers).  Pinned host sources copy
    asynchronously; the staging buffers are only rewritten after the previous staged batch has been consumed."""
    if self._stage is None:
      self._stage = dict(
          x=torch.empty_like(self.x), y=torch.empty_like(self.labels if self.labels is not None else self.labels_f),
          stream=torch.cuda.Stream(device=self.device), ready=torch.cuda.Event(), consumed=None)
    st = self._stage
    with torch.cuda.stream(st["stream"]):
      if st["consumed"] is not None:
        st["stream"].wait_event(st["consumed"])
      st["x"].copy_(torch.as_tensor(x).reshape(self.batch, self.in_dim), non_blocking=True)
      st["y"].copy_(torch.as_tensor(y).reshape(st["y"].shape), non_blocking=True)
      st["ready"].record(st["stream"])
    st["pending"] = True

  def _consume_staged(self):
    st = self._stage
    main = torch.cuda.current_stream(self.device)
    main.wait_event(st["ready"])
    self.x.copy_(st["x"], non_blocking=True)
    (self.labels if self.labels is not None else self.labels_f).copy_(st["y"], non_blocking=True)
    st["consumed"] = torch.cuda.Event()
    st["consumed"].record(main)
    st["pending"] = False

  # -- one step --------------------------------------------------------------
  def _fwd_waves(self, fwd, sp: int):
    """Layer waves: one grouped forward launch per layer index and distinct batch size, larger batches first.
    `fwd`: (net, input planes, batch, step counter of a TRAIN-mode forward or None, first minibatch row) per net."""
    for w in range(max((len(n.ws) for n, _, _, _, _ in fwd), default=0)):
      for bsz in sorted({b for _, _, b, _, _ in fwd}, reverse=True):
        ops = [n.fwd_op(w, xp, sd, r0) for n, xp, b, sd, r0 in fwd if b == bsz and w < len(n.ws)]
        if ops:
          _lib.check(self.lib.adn_dense_fwd_p_group((_lib.FwdOp * len(ops))(*ops), len(ops), bsz, sp),
                     "adn_dense_fwd_p_group")

  def _bwd_waves(self, cands, xp_of, sp: int):
    """Backward waves of the candidates, logits layer first: one grouped launch per wave and distinct batch size.
    `xp_of(c)`: the input planes of candidate c."""
    for k in range(max((len(c.net.ws) for c in cands), default=0)):
      for bsz in sorted({c.batch for c in cands}, reverse=True):
        ops = [c.bwd_op(k, xp_of(c)) for c in cands if c.batch == bsz and k < len(c.net.ws)]
        if ops:
          _lib.check(self.lib.adn_dense_bwd_p_group((_lib.BwdOp * len(ops))(*ops), len(ops), bsz, sp),
                     "adn_dense_bwd_p_group")

  def _enqueue_waves(self):
    """Plane path: layer waves across ALL subnetworks of the GPU (frozen members and candidates) as grouped
    launches on the main stream; the per-candidate small work (losses, ensemble heads, EMA / trace rows, optimizers)
    is grouped into one launch each (22 launches per step for 8 candidates); row-sharded candidates average their
    gradient arena across their ranks before the optimizer.  Bagged subnetworks take their own step first, through
    the same builders.  A rank without candidates only replays its frozen members."""
    lib = self.lib
    main = torch.cuda.current_stream(self.device)
    sp = main.cuda_stream
    # bagging pre-pass (adanet/autoensemble/common.py:43-56,151-180): a bagged subnetwork takes one training step
    # on a minibatch of its own input_fn BEFORE the main pass, which then only reads its (updated) forward
    bag = [c for c in self.candidates if c.bagged]
    if bag:
      for c in bag:
        if c.xp_own is not None:
          _lib.check(lib.adn_planes_split(c.x_own.data_ptr(), self.batch, c.net.in_dim, c.xp_own.data_ptr(), sp),
                     "adn_planes_split")
        else:
          c.net.stem_forward(lib, c.x_own, sp)
      self._fwd_waves([(c.net, c.xp_own, c.batch, self.step_dev, 0) for c in bag], sp)
      own = self.labels is not None
      ops = [c.sub_head_op(c.labels_own if own else None, None if own else c.labels_own, c.own_out3) for c in bag]
      _lib.check(lib.adn_head_group((_lib.HeadOp * len(ops))(*ops), len(ops), self.batch, self.C, sp), "adn_head_group")
      self._bwd_waves(bag, lambda c: c.xp_own, sp)
      for c in bag:
        if c.net.stem:
          c.enqueue_stem_bwd(c.x_own, sp)
      oops = [c.sub_opt.op(c._grads) for c in bag]
      _lib.check(lib.adn_opt_step_group((_lib.OptOp * len(oops))(*oops), len(oops), sp), "adn_opt_step_group")
    self._split_x(sp)
    # a row-sharded candidate consumes its own slice of the minibatch rows
    for c in self.sharded:
      if c.xp_local is not None:
        _lib.check(lib.adn_planes_split(self.x.data_ptr() + c.row0 * self.in_dim * 4, c.batch, self.in_dim,
                                        c.xp_local.data_ptr(), sp), "adn_planes_split")
    xp_of = lambda c: c.xp_local if c.xp_local is not None else self.xp
    x_of = lambda c: self.x[c.row0:c.row0 + c.batch] if c.comm is not None else self.x
    for f in self.frozen:
      if f.stem:
        f.stem_forward(lib, self.x, sp)
    for c in self.candidates:
      if c.net.stem:
        c.net.stem_forward(lib, x_of(c), sp)
    # whole candidates and frozen members run the full minibatch, row-sharded candidates their slice; candidates run
    # in TRAIN mode (dropout), a row-sharded one draws its rows of the whole minibatch's mask
    self._fwd_waves([(f, self.xp, self.batch, None, 0) for f in self.frozen] +
                    [(c.net, xp_of(c), c.batch, self.step_dev, c.row0) for c in self.candidates], sp)
    # steps 3 and 6-11 of every candidate in one grouped launch (+ one finalize): the subnetwork losses (dlogits planes,
    # logits-layer bias gradients) and every SCALAR / VECTOR candidate-ensemble head; MATRIX heads run their plane
    # GEMMs around their own head launch
    hops = [(c.sub_head_op(self.labels, self.labels_f, c.sub_out3), c.batch) for c in self.candidates]
    hops += [(h.head_op(self.labels, self.labels_f), h.batch) for _, h, _ in self.heads if h.groupable]
    for bsz in sorted({b for _, b in hops}, reverse=True):
      ops = [o for o, b in hops if b == bsz]
      _lib.check(lib.adn_head_group((_lib.HeadOp * len(ops))(*ops), len(ops), bsz, self.C, sp), "adn_head_group")
    for _, h, _ in self.heads:
      if not h.groupable:
        h.enqueue_matrix(self.labels, self.labels_f, sp, self.xp)
    trained = [c for c in self.candidates if not c.bagged]      # bagged subnetworks already took their step
    self._bwd_waves(trained, xp_of, sp)
    for c in trained:
      if c.net.stem:
        c.enqueue_stem_bwd(x_of(c), sp)
    # row-sharded candidates: ONE all-reduce (mean) per candidate of its gradient arena -- weight / bias gradients of
    # the slice, mixture-weight gradients and the loss scalars become those of the whole minibatch, bit-identical on
    # every rank of the candidate, so their replicas of the weights never diverge
    for c in self.sharded:
      c.comm.average_(c.arena.used())
    # steps 12-13: EMA and loss-trace row of every head, one launch
    books = [h.book() for _, h, _ in self.heads]
    if books:
      _lib.check(lib.adn_head_bookkeeping((_lib.HeadBook * len(books))(*books), len(books), self.step_dev.data_ptr(), sp),
                 "adn_head_bookkeeping")
    # steps 4-5 and 11 (apply): every optimizer of the step in one launch -- the mixture weights' (their gradients came
    # from the heads above; nothing read the weights since) and the subnetworks'
    oops = [h.ens_opt.op(h._ens_grads) for _, h, _ in self.heads if h.ens_opt is not None]
    oops += [c.sub_opt.op(c._grads) for c in trained]
    if oops:
      _lib.check(lib.adn_opt_step_group((_lib.OptOp * len(oops))(*oops), len(oops), sp), "adn_opt_step_group")
    _lib.check(lib.adn_counter_add(self.step_dev.data_ptr(), 1, sp), "adn_counter_add")

  def _enqueue(self):
    if self.xp is not None:
      return self._enqueue_waves()
    # fp32 SIMT cross-check: the frozen members' forward, then every candidate's whole step op by op on its own stream
    lib = self.lib
    main = torch.cuda.current_stream(self.device)
    sp = main.cuda_stream
    for f in self.frozen:   # shared by every candidate ensemble on this GPU
      f.forward(lib, self.x, sp)
    if self.multi_stream:
      for c, s in zip(self.candidates, self.streams):
        s.wait_stream(main)
        with torch.cuda.stream(s):
          c.enqueue_simt_step(self.x, self.labels, self.labels_f, self.step_dev, s.cuda_stream)
      for s in self.streams:
        main.wait_stream(s)
    else:
      for c in self.candidates:
        c.enqueue_simt_step(self.x, self.labels, self.labels_f, self.step_dev, sp)
    _lib.check(lib.adn_counter_add(self.step_dev.data_ptr(), 1, sp), "adn_counter_add")

  def _split_x(self, sp: int):
    # the minibatch's own planes feed first dense layers (and MATRIX weights of linear members); conv stems read x
    if self.xp is not None and any(not n.stem for n in list(self.frozen) + [c.net for c in self.candidates]):
      _lib.check(self.lib.adn_planes_split(self.x.data_ptr(), self.batch, self.in_dim, self.xp.data_ptr(), sp),
                 "adn_planes_split")

  def train_step(self, x=None, y=None, own_batches: Optional[Dict[int, tuple]] = None):
    """One training step of every candidate on this GPU on one minibatch: the one passed in, or the one
    started earlier with `stage_batch`.  `own_batches[candidate_index] = (x, y)` feeds the bagged subnetworks
    (those whose spec has `own_input`); each must get a fresh minibatch every step."""
    for c in self.candidates:
      if c.bagged:
        if own_batches is None or c.index not in own_batches:
          raise ValueError("bagged subnetwork %s needs its own minibatch (own_batches[%d])" % (c.spec.name, c.index))
        c.load_own_batch(*own_batches[c.index])
    if x is not None:
      self.load_batch(x, y)
    elif self._stage is not None and self._stage.get("pending"):
      self._consume_staged()
    if not self.use_cuda_graph or not self._warmed:
      # the plan's FIRST step always runs eagerly: every kernel variant of the step is launched (and lazily loaded by
      # the driver) once outside any stream capture -- a first launch inside the capture can invalidate it
      before = _lib.launch_count()
      self._enqueue()
      self.launches_per_step = _lib.launch_count() - before
      self._warmed = True
    else:
      if self._graph is None:
        import gc
        before = _lib.launch_count()
        g = torch.cuda.CUDAGraph()
        # graph capture records the launches without running them: no state changes.  The collector stays off while
        # the stream is capturing (destroying another plan's graph / events in the middle of it is not capture-safe).
        gc_was_on = gc.isenabled()
        gc.disable()
        try:
          with torch.cuda.graph(g):
            self._enqueue()
        finally:
          if gc_was_on:
            gc.enable()
        self.launches_per_step = _lib.launch_count() - before
        self._graph = g
      self._graph.replay()
    self.steps_done += 1

  def eval_step(self, x, y, metric: str = "adanet_loss") -> List[float]:
    """Forward-only metric of every local candidate ensemble on one hold-out batch of b <= batch examples (the
    Evaluator path, adanet/core/estimator.py:1469-1490): "adanet_loss" (default), "loss" / "average_loss" (the
    head's mean loss over the b examples) or "accuracy" (classification heads; arg-max of the ensemble logits,
    sigmoid heads at 0).  The members run in inference mode (no dropout) at the static batch, a partial batch
    zero-padded; the heads read the first b rows."""
    if metric not in EVAL_METRICS:
      raise NotImplementedError("Evaluator metric %r is not computed by the B200 engine (supported: %s)" % (metric, ", ".join(EVAL_METRICS)))
    if metric == "accuracy" and self.head == "mse":
      raise ValueError("accuracy is not an evaluation metric of a regression head")
    if self.sharded:
      raise NotImplementedError("hold-out evaluation of row-sharded candidates: use placement='balanced' with an Evaluator")
    labels = self.labels if self.labels is not None else self.labels_f
    b = _load_rows(self.x, labels, x, y)
    sp = torch.cuda.current_stream(self.device).cuda_stream
    self._split_x(sp)
    for f in self.frozen:
      f.forward(self.lib, self.x, sp, self.xp)
    for c in self.candidates:
      c.net.forward(self.lib, self.x, sp, self.xp)
    out = []
    ens_out = torch.empty((self.batch, self.C), dtype=torch.float32, device=self.device) if metric == "accuracy" else None
    for _, h, _ in self.heads:
      h.enqueue_eval(self.labels, self.labels_f, ens_out, sp, self.xp, rows=b)
      if metric == "accuracy":
        out.append(accuracy_of(ens_out[:b], labels[:b]))
    torch.cuda.current_stream(self.device).synchronize()
    if metric == "accuracy":
      return out
    return [float(h.out3[2 if metric == "adanet_loss" else 0].item()) for _, h, _ in self.heads]

  # -- in-flight checkpoint -------------------------------------------------------
  def state_dict(self) -> Dict[str, np.ndarray]:
    """State of the iteration in flight on this GPU (one flat dict, keys prefixed by candidate index)."""
    torch.cuda.current_stream(self.device).synchronize()
    out = {"steps_done": np.asarray(self.steps_done, dtype=np.int64), "step_dev": self.step_dev.cpu().numpy()}
    for c in self.candidates:
      for k, v in c.state_dict().items():
        out["c%d_%s" % (c.index, k)] = v
    for gidx, h, _ in self.heads:
      if not any(h is c.ehead for c in self.candidates):
        for k, v in h.state_dict().items():
          out["h%d_%s" % (gidx, k)] = v
    return out

  def load_state_dict(self, st: Dict[str, np.ndarray]):
    self.steps_done = int(st["steps_done"])
    self.step_dev.copy_(torch.as_tensor(st["step_dev"]))
    for c in self.candidates:
      pre = "c%d_" % c.index
      c.load_state_dict({k[len(pre):]: v for k, v in st.items() if k.startswith(pre)})
    for gidx, h, _ in self.heads:
      if not any(h is c.ehead for c in self.candidates):
        pre = "h%d_" % gidx
        h.load_state_dict({k[len(pre):]: v for k, v in st.items() if k.startswith(pre)})
    torch.cuda.current_stream(self.device).synchronize()

  def plane_overflow(self, reset: bool = True) -> bool:
    """True when a finite value did not fit the fp16 planes since the flag was last read (csrc/plane_fmt.cuh), or the
    in-flight state this plan resumed from was saved after one (`carried_overflow`); the caller re-runs the iteration
    on TF32 planes (AdaNetSearch.run / Estimator.train)."""
    if self.fmt != _lib.PLANES_F16 or self.xp is None:
      return False
    return _lib.plane_overflow(torch.cuda.current_stream(self.device).cuda_stream, reset) or self.carried_overflow

  # -- read-back ---------------------------------------------------------------
  def _reports(self, h) -> bool:
    """A row-sharded candidate's head exists on every rank of its group; only the first one reports it."""
    c = next((c for c in self.sharded if c.ehead is h), None)
    return c is None or c.comm.index == 0

  def ema_losses(self) -> List[float]:
    """EMA adanet loss of each local candidate this rank reports (candidate.py:125-129), one D2H read."""
    torch.cuda.current_stream(self.device).synchronize()
    return [float(h.ema_state[2].item()) for _, h, _ in self.heads if self._reports(h)]

  def traces(self) -> Dict[str, Dict[str, np.ndarray]]:
    """Per-step (sub_loss, ens_loss, adanet_loss, ema) of every head over the last min(steps_done, trace_capacity)
    steps, oldest first.  Step s writes row s % trace_capacity of the ring, so once it has wrapped the oldest kept
    step sits at row steps_done % trace_capacity."""
    n = min(self.steps_done, self.trace_capacity)
    order = (np.arange(self.steps_done - n, self.steps_done) % self.trace_capacity) if n else np.zeros((0,), np.int64)
    out = {}
    for _, h, _ in self.heads:
      t = h.trace.cpu().numpy()[order]
      out[h.name] = {f: t[:, i].copy() for i, f in enumerate(TRACE_FIELDS)}
    return out

  def last_losses(self) -> np.ndarray:
    """[n_candidates, 4] (sub_loss, ens_loss, adanet_loss, ema) of the most recent step."""
    row = (self.steps_done - 1) % self.trace_capacity
    return torch.stack([h.trace[row] for _, h, _ in self.heads]).cpu().numpy()


class EnsembleEvalPlan:
  """Forward-only evaluation of a finished ensemble (evaluate / predict and the
  `previous_ensemble` candidate of the Evaluator): frozen members replayed with
  adn_dense_fwd, then adn_ensemble_head for logits and loss
  (adanet/core/estimator.py:1785-1882 rebuilds the same thing as a TF graph)."""

  def __init__(self, members: Sequence[DenseNet], mix_w: np.ndarray, bias: np.ndarray, ens: EnsemblerPlanSpec,
               head: str, batch: int, logits_dim: int, device: Optional[torch.device] = None):
    self.lib = _require_cuda()
    self.device = device or torch.device("cuda", torch.cuda.current_device())
    self.members, self.batch, self.C, self.head = list(members), batch, logits_dim, _HEAD_KIND[head]
    self.fmt = _lib.plane_format()      # xp / mwp are sized for it: a plan outlives no format switch
    for m in self.members:
      m.ensure_format()
      if m.batch != batch:
        raise ValueError("member %s was built for batch %d, eval plan uses %d" % (m.name, m.batch, batch))
    f32 = dict(dtype=torch.float32, device=self.device)
    self.mix = _MIX_KIND[ens.mixture_weight_type]
    if self.mix == _lib.MIX_MATRIX:
      # mix_w: list of [D_k, C] matrices; members are pre-multiplied by the plane GEMM, w = their L1 norms
      if not planes_enabled():
        raise NotImplementedError("MATRIX mixture weights run on the plane path only")
      self.mw = [torch.as_tensor(np.ascontiguousarray(w, dtype=np.float32)).to(self.device) for w in mix_w]
      self.mwp = [new_planes(w.shape[0], w.shape[1], self.device) for w in self.mw]
      sp0 = torch.cuda.current_stream(self.device).cuda_stream
      for w, wp in zip(self.mw, self.mwp):
        _lib.check(self.lib.adn_planes_split(w.data_ptr(), w.shape[0], w.shape[1], wp.data_ptr(), sp0), "adn_planes_split")
      self.mw_logits = [torch.empty((batch, logits_dim), **f32) for _ in self.mw]
      self.mix_w = torch.as_tensor(np.array([np.abs(np.asarray(w, dtype=np.float32)).sum(dtype=np.float32)
                                             for w in mix_w], dtype=np.float32)).to(self.device)
    else:
      self.mix_w = torch.as_tensor(np.ascontiguousarray(mix_w, dtype=np.float32)).to(self.device).reshape(
          (len(members),) if self.mix == _lib.MIX_SCALAR else (len(members), logits_dim))
    self.bias = torch.as_tensor(np.ascontiguousarray(bias, dtype=np.float32)).to(self.device)
    lam, beta = float(ens.adanet_lambda), float(ens.adanet_beta)
    self.reg_is_zero = int(lam == 0.0 and beta == 0.0)
    self.gammas = gammas(lam, beta, [m.complexity for m in self.members])
    self._gammas = _lib.f32_array(self.gammas)
    self._members = _lib.ptr_array([t.data_ptr() for t in self.mw_logits] if self.mix == _lib.MIX_MATRIX
                                   else [m.logits.data_ptr() for m in self.members])
    self.out3 = torch.zeros((3,), **f32)
    self.ens_logits = torch.empty((batch, logits_dim), **f32)
    self.rows = 0             # examples of the last `run`: its logits are the first rows of ens_logits
    self.ws_bytes = _lib.query(_lib.Q_HEAD_WS, batch, logits_dim, len(self.members))
    self.workspace = torch.empty((self.ws_bytes,), dtype=torch.uint8, device=self.device)
    self.x = torch.empty((batch, members[0].in_dim), **f32)
    self.xp = new_planes(batch, members[0].in_dim, self.device) if planes_enabled() else None
    self.labels = torch.zeros((batch,), dtype=torch.int64, device=self.device) if head == "softmax_xent" else None
    self.labels_f = torch.zeros((batch, logits_dim), **f32) if head != "softmax_xent" else None

  def run(self, x, y=None, forward_members: bool = True):
    """Evaluates the ensemble on the b <= batch examples of `x`: returns (loss, reg, adanet_loss) over them as
    floats (NaN-free only when labels given) and leaves their ensemble logits in the first b rows of
    `self.ens_logits` (`self.rows` = b).  The members run at the static batch, a partial batch zero-padded."""
    sp = torch.cuda.current_stream(self.device).cuda_stream
    b = _load_rows(self.x, self.labels if self.labels is not None else self.labels_f, x, y)
    self.rows = b
    _check_head_ws(b, self.C, len(self.members), self.ws_bytes)
    if forward_members:
      if self.xp is not None and any(not m.stem for m in self.members):
        _lib.check(self.lib.adn_planes_split(self.x.data_ptr(), self.batch, self.x.shape[1], self.xp.data_ptr(), sp),
                   "adn_planes_split")
      for m in self.members:
        m.forward(self.lib, self.x, sp, self.xp)
      if self.mix == _lib.MIX_MATRIX:
        matrix_member_logits(self.lib, self.members, self.mwp, self.mw_logits, self.xp, sp)
    _lib.check(self.lib.adn_ensemble_head(
        self.head, self.mix, self._members, len(self.members), self.mix_w.data_ptr(), self.bias.data_ptr(),
        self._gammas, self.reg_is_zero, 1.0, self.labels.data_ptr() if self.labels is not None else None,
        self.labels_f.data_ptr() if self.labels_f is not None else None, self.out3.data_ptr(), None, None, None,
        self.ens_logits.data_ptr(), b, self.C, self.workspace.data_ptr(), self.ws_bytes, sp),
               "adn_ensemble_head")
    o = self.out3.cpu().numpy()
    return float(o[0]), float(o[1]), float(o[2])

  def metric(self, x, y, metric: str = "adanet_loss") -> float:
    """One Evaluator metric of the finished ensemble on a batch (see IterationPlan.eval_step)."""
    if metric not in EVAL_METRICS:
      raise NotImplementedError("Evaluator metric %r is not computed by the B200 engine (supported: %s)" % (metric, ", ".join(EVAL_METRICS)))
    loss, _, adanet = self.run(x, y)
    if metric == "accuracy":
      if self.head == _lib.HEAD_MSE:
        raise ValueError("accuracy is not an evaluation metric of a regression head")
      b = self.rows
      return accuracy_of(self.ens_logits[:b], (self.labels if self.labels is not None else self.labels_f)[:b])
    return adanet if metric == "adanet_loss" else loss
