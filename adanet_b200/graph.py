"""A tiny symbolic graph: what `Builder.build_subnetwork` constructs here.

The reference's builders create TF1 graph tensors (`tf.layers.dense`,
`feature_column.input_layer`, `tf.nn.relu`, `tf.layers.dropout`;
adanet/examples/simple_dnn.py:61-101) that TensorFlow later executes.  The
B200 engine executes dense subnetworks with its own CUDA kernels, so builders
describe the computation with the same *vocabulary* over symbolic handles; the
Estimator lowers the finished graph to an engine plan
(adanet_b200/core/lowering.py).  Only the hot path's vocabulary exists: a
builder that needs an op outside it gets a clear NotImplementedError at build
time, never a silent CPU fallback.
"""

from __future__ import annotations

import contextlib
import math
from typing import Dict, Iterable, List, Optional, Sequence

import numpy as np


class Variable:
  """A trainable parameter with its initial value (tf.Variable stand-in)."""

  def __init__(self, name: str, value: np.ndarray, trainable: bool = True):
    self.name, self.value, self.trainable = name, np.asarray(value, dtype=np.float32), trainable

  def __repr__(self):
    return "Variable(%s, shape=%s)" % (self.name, self.value.shape)


class Tensor:
  """Symbolic tensor: static shape (batch dimension None) + producing op."""

  def __init__(self, shape: Sequence[Optional[int]], op: str, inputs: Sequence["Tensor"] = (), attrs: Optional[dict] = None,
               name: Optional[str] = None):
    self.shape, self.op, self.inputs, self.attrs, self.name = tuple(shape), op, tuple(inputs), dict(attrs or {}), name

  def get_shape(self):
    return self

  def as_list(self):
    return list(self.shape)

  def __repr__(self):
    return "Tensor(op=%s, shape=%s)" % (self.op, self.shape)


class Graph:
  """Collects the variables a builder creates (the `var_list` of
  adanet/core/ensemble_builder.py:224-255,754 is a collection diff)."""

  def __init__(self):
    self.variables: List[Variable] = []
    self._names: Dict[str, int] = {}

  def unique_name(self, base: str) -> str:
    n = self._names.get(base, 0)
    self._names[base] = n + 1
    return base if n == 0 else "%s_%d" % (base, n)

  def add(self, v: Variable):
    self.variables.append(v)


_graph_stack: List[Graph] = [Graph()]


def get_default_graph() -> Graph:
  return _graph_stack[-1]


@contextlib.contextmanager
def graph_scope():
  g = Graph()
  _graph_stack.append(g)
  try:
    yield g
  finally:
    _graph_stack.pop()


# ---------------------------------------------------------------------------
# initializers
# ---------------------------------------------------------------------------


def glorot_uniform_initializer(seed: Optional[int] = None):
  """U(-l, l), l = sqrt(6/(fan_in+fan_out)) [TF glorot_uniform].  NumPy's
  generator, not TF's Philox stream: parity runs inject weights instead."""
  state = {"rng": np.random.default_rng(seed)}

  def init(shape):
    fan_in, fan_out = shape[0], shape[-1]
    limit = math.sqrt(6.0 / (fan_in + fan_out))
    return state["rng"].uniform(-limit, limit, size=shape).astype(np.float32)

  return init


def he_normal_initializer(seed: Optional[int] = None):
  """tf.keras.initializers.he_normal [TF]: VarianceScaling(scale=2, mode="fan_in", truncated normal), i.e.
  N(0, sqrt(2/fan_in)/0.8796...) truncated at two standard deviations; fan_in = prod(shape[:-1])
  (9*Cin for a 3x3 conv kernel, `in` for a dense kernel).  NumPy's generator, not TF's stream."""
  state = {"rng": np.random.default_rng(seed)}

  def init(shape):
    fan_in = int(np.prod(shape[:-1]))
    std = math.sqrt(2.0 / max(1, fan_in)) / 0.87962566103423978
    rng = state["rng"]
    out = rng.standard_normal(shape)
    bad = np.abs(out) > 2.0
    while bad.any():                       # resample the tails (truncated normal)
      out[bad] = rng.standard_normal(int(bad.sum()))
      bad = np.abs(out) > 2.0
    return (out * std).astype(np.float32)

  return init


def zeros_initializer():
  return lambda shape: np.zeros(shape, dtype=np.float32)


def constant_initializer(value):
  """Injects explicit initial values (array) or a scalar fill."""
  def init(shape):
    v = np.asarray(value, dtype=np.float32)
    if v.shape == tuple(shape):
      return v.copy()
    if v.ndim == 0:
      return np.full(shape, float(v), dtype=np.float32)
    raise ValueError("constant_initializer: value shape %s does not match variable shape %s" % (v.shape, tuple(shape)))
  return init


# ---------------------------------------------------------------------------
# feature columns and ops
# ---------------------------------------------------------------------------


class NumericColumn:
  """feature_column.numeric_column(key, shape) [TF]."""

  def __init__(self, key: str, shape=(1,)):
    self.key = key
    self.shape = (shape,) if isinstance(shape, int) else tuple(shape)
    self.name = key

  @property
  def width(self) -> int:
    return int(np.prod(self.shape))


def numeric_column(key: str, shape=(1,)) -> NumericColumn:
  return NumericColumn(key, shape)


def placeholder(width, name: str) -> Tensor:
  """A fed tensor [batch, width], or [batch, *shape] when `width` is a shape tuple (NHWC images)."""
  shape = (None, int(width)) if np.ndim(width) == 0 else (None,) + tuple(int(v) for v in width)
  return Tensor(shape, "placeholder", (), {"key": name}, name)


def input_layer(features, feature_columns: Iterable[NumericColumn]) -> Tensor:
  """feature_column.input_layer [TF]: numeric columns concatenated in sorted-name
  order (adanet/examples/simple_dnn.py:70-71)."""
  cols = sorted(feature_columns, key=lambda c: c.name)
  if not cols:
    raise ValueError("feature_columns must not be empty")
  if isinstance(features, Tensor):
    features = {cols[0].key: features} if len(cols) == 1 else None
  if not isinstance(features, dict):
    raise ValueError("features must be a dict of column key -> Tensor")
  parts = []
  for c in cols:
    if c.key not in features:
      raise ValueError("Feature %s is not in features dictionary." % c.key)
    t = features[c.key]
    if t.shape[-1] != c.width:
      raise ValueError("feature %s has width %s, column expects %d" % (c.key, t.shape[-1], c.width))
    parts.append(t)
  width = sum(p.shape[-1] for p in parts)
  return Tensor((None, width), "input_layer", parts, {"keys": [c.key for c in cols]})


def relu(x: Tensor) -> Tensor:
  return Tensor(x.shape, "relu", (x,))


def concat(values: Sequence[Tensor], axis: int = -1) -> Tensor:
  """tf.concat [TF] of rank-2 tensors [batch, width] on the last axis: what a builder uses to read the hidden layers
  of previous-iteration subnetworks (adanet/core/estimator_test.py _DNNBuilder).  The engine lowers a dense layer over
  it to one GEMM over the pieces (core/lowering.py); any other axis or rank raises NotImplementedError."""
  values = list(values)
  if not values or not all(isinstance(v, Tensor) for v in values):
    raise ValueError("concat expects a non-empty list of Tensors, got %r" % (values,))
  ranks = {len(v.shape) for v in values}
  if len(ranks) != 1:
    raise ValueError("concat of tensors of different ranks: %s" % ([v.shape for v in values],))
  rank = ranks.pop()
  if rank != 2:
    raise NotImplementedError("concat is implemented for rank-2 tensors [batch, width] (got rank %d)" % rank)
  if not -rank <= axis < rank:
    raise ValueError("concat axis %d is out of range for rank-2 tensors" % axis)
  if axis % rank != rank - 1:
    raise NotImplementedError("concat is implemented on the last axis only (got axis=%d)" % axis)
  batch = {v.shape[0] for v in values} - {None}
  if len(batch) > 1:
    raise ValueError("concat of tensors with different batch dimensions: %s" % ([v.shape for v in values],))
  return Tensor((batch.pop() if batch else None, sum(int(v.shape[-1]) for v in values)), "concat", values)


def dense(inputs: Tensor, units: int, activation=None, use_bias: bool = True, kernel_initializer=None,
          bias_initializer=None, name: Optional[str] = None) -> Tensor:
  """tf.layers.dense [TF]: kernel [in, units] (default glorot-uniform), bias zeros."""
  if activation not in (None, relu, "relu"):
    raise NotImplementedError("adanet_b200 dense layers support activation None or relu (got %r)" % (activation,))
  g = get_default_graph()
  in_dim = inputs.shape[-1]
  base = g.unique_name(name or "dense")
  kinit = kernel_initializer or glorot_uniform_initializer()
  kernel = Variable(base + "/kernel", kinit((in_dim, units)))
  g.add(kernel)
  bias = None
  if use_bias:
    bias = Variable(base + "/bias", (bias_initializer or zeros_initializer())((units,)))
    g.add(bias)
  return Tensor((None, units), "dense", (inputs,),
                {"kernel": kernel, "bias": bias, "activation": "relu" if activation is not None else None}, base)


def conv2d(inputs: Tensor, filters: int, kernel_size=3, strides=1, padding: str = "valid", activation=None,
           use_bias: bool = True, kernel_initializer=None, bias_initializer=None, name: Optional[str] = None) -> Tensor:
  """tf.keras.layers.Conv2D / tf.layers.conv2d [TF] on NHWC images: kernel [kh, kw, Cin, filters] (HWIO).
  The engine runs the SimpleCNN stem -- 3x3, stride 1, padding "same", ReLU -- and nothing else (csrc/conv_stem.cu)."""
  ks = (kernel_size, kernel_size) if np.ndim(kernel_size) == 0 else tuple(kernel_size)
  st = (strides, strides) if np.ndim(strides) == 0 else tuple(strides)
  if len(inputs.shape) != 4:
    raise ValueError("conv2d expects NHWC images [batch, H, W, C], got shape %s" % (inputs.shape,))
  if ks != (3, 3) or st != (1, 1) or str(padding).lower() != "same":
    raise NotImplementedError("the B200 engine implements conv2d with kernel_size=3, strides=1, padding='same' "
                              "(got kernel_size=%s strides=%s padding=%r)" % (ks, st, padding))
  if activation not in (None, relu, "relu"):
    raise NotImplementedError("conv2d supports activation None or relu (got %r)" % (activation,))
  g = get_default_graph()
  _, h, w, cin = inputs.shape
  base = g.unique_name(name or "conv2d")
  kernel = Variable(base + "/kernel", (kernel_initializer or glorot_uniform_initializer())((3, 3, cin, filters)))
  g.add(kernel)
  bias = None
  if use_bias:
    bias = Variable(base + "/bias", (bias_initializer or zeros_initializer())((filters,)))
    g.add(bias)
  return Tensor((None, h, w, filters), "conv2d", (inputs,),
                {"kernel": kernel, "bias": bias, "activation": "relu" if activation is not None else None}, base)


def max_pooling2d(inputs: Tensor, pool_size=2, strides=2, padding: str = "valid") -> Tensor:
  """tf.keras.layers.MaxPool2D [TF]; the engine fuses the 2x2 / stride 2 pool into the conv stem."""
  ps = (pool_size, pool_size) if np.ndim(pool_size) == 0 else tuple(pool_size)
  st = (strides, strides) if np.ndim(strides) == 0 else tuple(strides)
  if len(inputs.shape) != 4:
    raise ValueError("max_pooling2d expects [batch, H, W, C], got shape %s" % (inputs.shape,))
  if ps != (2, 2) or st != (2, 2):
    raise NotImplementedError("the B200 engine implements max pooling with pool_size=2, strides=2")
  _, h, w, c = inputs.shape
  if h % 2 or w % 2:
    raise NotImplementedError("max_pooling2d needs even height and width (got %dx%d)" % (h, w))
  return Tensor((None, h // 2, w // 2, c), "max_pool2d", (inputs,))


def flatten(inputs: Tensor) -> Tensor:
  """tf.keras.layers.Flatten [TF]: [batch, ...] -> [batch, prod(...)] in row-major (h, w, c) order."""
  return Tensor((None, int(np.prod(inputs.shape[1:]))), "flatten", (inputs,))


class layers:
  """Keras-style spellings of the ops above, so a builder written against `tf.keras.layers`
  (customizing_adanet.ipynb SimpleCNNBuilder) keeps its shape: `layers.Conv2D(...)(images)`."""

  class Conv2D:
    def __init__(self, filters, kernel_size, strides=1, padding="valid", activation=None, use_bias=True,
                 kernel_initializer=None, bias_initializer=None, name=None):
      self._kw = dict(filters=filters, kernel_size=kernel_size, strides=strides, padding=padding, activation=activation,
                      use_bias=use_bias, kernel_initializer=kernel_initializer, bias_initializer=bias_initializer, name=name)

    def __call__(self, inputs):
      return conv2d(inputs, **self._kw)

  class MaxPool2D:
    def __init__(self, pool_size=2, strides=None, padding="valid"):
      self._kw = dict(pool_size=pool_size, strides=pool_size if strides is None else strides, padding=padding)

    def __call__(self, inputs):
      return max_pooling2d(inputs, **self._kw)

  class Flatten:
    def __call__(self, inputs):
      return flatten(inputs)

  class Dense:
    def __init__(self, units, activation=None, use_bias=True, kernel_initializer=None, bias_initializer=None, name=None):
      self._kw = dict(units=units, activation=activation, use_bias=use_bias, kernel_initializer=kernel_initializer,
                      bias_initializer=bias_initializer, name=name)

    def __call__(self, inputs):
      return dense(inputs, **self._kw)


def dropout(inputs: Tensor, rate: float = 0.0, seed=None, training: bool = False) -> Tensor:
  """tf.layers.dropout (adanet/examples/simple_dnn.py:80-81): identity unless training with rate > 0; then
  `inputs * keep_mask / (1 - rate)`.  The engine draws keep_mask from a counter-based hash of (seed, layer, step,
  element) in the epilogue of the layer that produces `inputs` (csrc/planes.cu emit_slice_fwd_planes; TF's own random
  stream is not reproduced -- the mask is injected data, like the initial weights)."""
  if not (training and rate and rate > 0.0):
    return inputs
  if not (0.0 < float(rate) < 1.0):
    raise ValueError("dropout rate must be in [0, 1), got %r" % (rate,))
  return Tensor(inputs.shape, "dropout", (inputs,), {"rate": float(rate), "seed": int(seed) if seed is not None else 0})


class Loss(Tensor):
  """Scalar head loss on some logits (what Builder.build_subnetwork_train_op receives)."""

  def __init__(self, logits: Tensor, kind: str):
    super().__init__((), "loss", (logits,), {"kind": kind})
