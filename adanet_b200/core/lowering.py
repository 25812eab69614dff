"""Lowers a Builder's symbolic Subnetwork to an engine plan spec.

The reference calls `builder.build_subnetwork(...)` inside a TF variable scope
and diffs the variable collections to find the builder's own variables
(adanet/core/ensemble_builder.py:679-805, var_list isolation :224-255,754);
then `builder.build_subnetwork_train_op(subnetwork, loss, var_list, ...)`.
Here the same two calls are made against the symbolic graph of
adanet_b200.graph, and the result -- a chain
input_layer -> [dense+relu]* -> dense -- becomes a SubnetworkPlanSpec.
"""

from __future__ import annotations

import inspect
from typing import Dict, List, Optional, Tuple

import numpy as np

from adanet_b200 import _lib
from adanet_b200 import graph
from adanet_b200 import subnetwork as subnetwork_lib
from adanet_b200 import train
from adanet_b200.core import engine as eng


class _NullSummary:
  """Stand-in for adanet.Summary (adanet/core/summary.py): TensorBoard plumbing is out of scope."""

  def scalar(self, name, tensor=None, family=None, **kwargs):
    return None

  image = audio = histogram = scalar

  def current_scope(self):
    import contextlib
    return contextlib.nullcontext()


def call_build_subnetwork(builder, features, labels, logits_dimension, training, iteration_step, summary,
                          previous_ensemble, config=None):
  """Calls build_subnetwork with `labels` / `config` only when the override declares them
  (argument-name sniffing, adanet/core/ensemble_builder.py:737-746)."""
  args = inspect.signature(builder.build_subnetwork).parameters
  kwargs = dict(features=features, logits_dimension=logits_dimension, training=training,
                iteration_step=iteration_step, summary=summary, previous_ensemble=previous_ensemble)
  if "labels" in args:
    kwargs["labels"] = labels
  if "config" in args:
    kwargs["config"] = config
  return builder.build_subnetwork(**kwargs)


# Every dense op of a lowered chain is stamped with attrs[_LAYER] = (iteration, builder name, layer index, is logits):
# a later iteration's builder that reads it (through previous_ensemble) names that member's layer.  Checkpoints
# restore such tensors as "member_layer" handles (attrs["ref"] = (iteration, name, layer)) and the input features a
# member read as an "input_ref" handle.
_LAYER = "adanet_layer"


def _member_piece(t: graph.Tensor, members) -> dict:
  """The piece a tensor from outside this subnetwork resolves to: a previous-iteration member's hidden layer, or the
  input features.  A relu or dropout wrapper names the same layer (member layers are ReLU outputs, and frozen members
  replay without dropout).  `members`: the (iteration, name) of the members it may read, or None for any."""
  wrapped = t.op in ("relu", "dropout")
  while t.op in ("relu", "dropout"):
    t = t.inputs[0]
  if t.op in ("input_layer", "input_ref"):
    if wrapped:
      raise NotImplementedError("relu or dropout on the input features inside a concat is not implemented by the B200 "
                                "engine")
    return {"src": "input"}
  if t.op == "member_layer":
    it, name, j = t.attrs["ref"]
    if t.attrs.get("is_logits"):
      raise NotImplementedError("the logits of subnetwork %s (iteration %d) cannot be read by another subnetwork: only "
                                "its hidden layers can" % (name, it))
  elif t.op == "dense" and _LAYER in t.attrs:
    it, name, j, is_logits = t.attrs[_LAYER]
    if is_logits:
      raise NotImplementedError("the logits of subnetwork %s (iteration %d) cannot be read by another subnetwork: only "
                                "its hidden layers can" % (name, it))
  elif t.op in ("flatten", "max_pool2d", "conv2d") or (t.op == "placeholder" and len(t.shape) == 4):
    raise NotImplementedError("a conv-stem output or the images cannot be a piece of a concat (op %r)" % t.op)
  elif t.op == "placeholder":
    raise NotImplementedError("a concat piece must be graph.input_layer(features, columns) or a subnetwork layer, not "
                              "the raw placeholder %r" % (t.name,))
  else:
    raise NotImplementedError("op %r cannot be a piece of a concat that a dense layer reads" % t.op)
  if members is not None and (int(it), name) not in members:
    raise NotImplementedError("subnetwork %s of iteration %d is not a member of the previous ensemble: a subnetwork "
                              "can only read the hidden layers of the previous ensemble's members" % (name, it))
  return {"src": "member", "iteration": int(it), "name": name, "layer": int(j)}


def _flatten_concat(t: graph.Tensor, relu: bool, out: list):
  """Nested concats flatten into one list of (tensor, under a relu(concat(...))) in concat order."""
  if t.op == "relu" and t.inputs[0].op == "concat":
    _flatten_concat(t.inputs[0], True, out)
  elif t.op == "concat":
    for v in t.inputs:
      _flatten_concat(v, relu, out)
  else:
    out.append((t, relu))


def _is_own(t: graph.Tensor) -> bool:
  while t.op in ("relu", "dropout"):
    t = t.inputs[0]
  return t.op == "dense" and _LAYER not in t.attrs


def _own_piece(t: graph.Tensor, relu: bool) -> graph.Tensor:
  """A concat element from this subnetwork's own chain: [dropout <-] [relu <-] dense.  Returns the dense op with its
  activation / dropout set; relu(concat(...)) folds into a linear dense the same way relu(dense) does."""
  drop = None
  if t.op == "dropout":
    drop, t = (t.attrs["rate"], t.attrs["seed"]), t.inputs[0]
  if t.op == "relu":
    t, relu = t.inputs[0], True
    if t.attrs.get("activation") is not None:
      raise NotImplementedError("relu must directly follow a linear dense layer")
  if t.op != "dense":
    raise NotImplementedError("op %r cannot be a piece of a concat that a dense layer reads" % t.op)
  if relu:
    if t.attrs.get("activation") is not None:
      raise NotImplementedError("relu(concat(...)) over a dense layer that already has an activation")
    t.attrs["activation"] = "relu"
  if drop is not None:
    t.attrs["dropout_after"] = drop
  return t


def _concat_pieces(t: graph.Tensor, members, name: str):
  """The pieces of a dense layer that reads concat `t` (or relu(concat)): (pieces in concat order, each with its
  width, and the tensor the chain continues from -- this subnetwork's own previous dense layer, or the input
  features when the layer is the first)."""
  elems = []
  _flatten_concat(t, False, elems)
  pieces, own, inputs = [], [], []
  for e, relu in elems:
    if _is_own(e):
      own.append(len(pieces))
      pieces.append(({"src": "own"}, _own_piece(e, relu)))
      continue
    p = _member_piece(e, members)
    if relu and p["src"] == "input":
      raise NotImplementedError("relu(concat(...)) over the input features")
    if p["src"] == "input":
      inputs.append(len(pieces))
    pieces.append((p, e))
  if len(own) > 1:
    raise NotImplementedError("subnetwork %s reads one of its own earlier hidden layers again: skip connections inside "
                              "one subnetwork are not implemented by the B200 engine" % name)
  if own:
    nxt = pieces[own[0]][1]
  elif inputs:
    # the first layer: the (first) input-features piece is its primary one, any other one is a dW-only piece
    pieces[inputs[0]] = ({"src": "own"}, pieces[inputs[0]][1])
    nxt = pieces[inputs[0]][1]
    while nxt.op in ("relu", "dropout"):
      nxt = nxt.inputs[0]
  else:
    raise NotImplementedError("a dense layer of subnetwork %s reads only hidden layers of other subnetworks: every layer "
                              "must read its own previous layer (the first one: the input features)" % name)
  if len(pieces) > 1 + _lib.FWD_MAX_SRCS:
    raise NotImplementedError("a dense layer of subnetwork %s reads %d pieces; the B200 engine runs at most %d (its "
                              "own previous layer and %d more)" % (name, len(pieces), 1 + _lib.FWD_MAX_SRCS,
                                                                   _lib.FWD_MAX_SRCS))
  out, r = [], 0
  for p, e in pieces:
    w = int(e.shape[-1])
    out.append(dict(p, rows=[r, r + w]))
    r += w
  return out, nxt


def _trace_dense_chain(logits: graph.Tensor, members=None, name: str = "") -> Tuple[List[graph.Tensor], graph.Tensor, list]:
  """Walks logits back to the input layer; returns (dense ops first->last, input tensor, pieces per layer: the
  resolved piece list of a layer over a concat, else None)."""
  chain, pieces = [], []
  t = logits
  pending_dropout = None
  while True:
    if t.op == "concat" or (t.op == "relu" and t.inputs[0].op == "concat"):
      if pending_dropout is not None or not chain:
        raise NotImplementedError("a concat must be read by a dense layer (no dropout between them)")
      ps, t = _concat_pieces(t, members, name)
      pieces[-1] = ps if len(ps) > 1 else None
      if t.op != "dense":
        break
    elif t.op == "dropout":
      # tf.layers.dropout on a hidden activation: belongs to the dense layer that produces it
      if pending_dropout is not None or not chain:
        raise NotImplementedError("dropout must follow a hidden dense+relu layer (one dropout per layer)")
      pending_dropout = (t.attrs["rate"], t.attrs["seed"])
      t = t.inputs[0]
    elif t.op == "dense":
      if _LAYER in t.attrs:
        raise NotImplementedError("a dense layer of subnetwork %s reads a layer of another subnetwork directly: read it "
                                  "through graph.concat next to the layer's own input" % name)
      pieces.append(None)
      if pending_dropout is not None:
        t.attrs["dropout_after"] = pending_dropout
        pending_dropout = None
      chain.append(t)
      t = t.inputs[0]
    elif t.op == "relu":
      # explicit relu(dense(...)) is folded into the dense's activation
      inner = t.inputs[0]
      if inner.op != "dense" or inner.attrs.get("activation") is not None:
        raise NotImplementedError("relu must directly follow a linear dense layer")
      inner.attrs["activation"] = "relu"
      t = inner
    elif t.op in ("input_layer", "placeholder", "flatten"):
      if pending_dropout is not None:
        raise NotImplementedError("dropout on the input features is not implemented by the B200 engine")
      break
    else:
      raise NotImplementedError(
          "the B200 engine runs dense subnetworks (input_layer -> [dense+relu]* -> dense), optionally behind a "
          "conv3x3+relu -> maxpool2 -> flatten stem; op %r is not supported" % t.op)
  chain.reverse()
  pieces.reverse()
  return chain, t, pieces


def _trace_conv_stem(flat: graph.Tensor):
  """flatten <- max_pool2d(2,2) <- [relu <-] conv2d(3x3, same) <- NHWC images: the SimpleCNN stem
  (customizing_adanet.ipynb SimpleCNNBuilder.build_subnetwork).  Returns (conv op, image placeholder)."""
  pool = flat.inputs[0]
  if pool.op != "max_pool2d":
    raise NotImplementedError("flatten must follow max_pooling2d in a conv-stem subnetwork (got op %r)" % pool.op)
  conv = pool.inputs[0]
  if conv.op == "relu":
    inner = conv.inputs[0]
    if inner.op != "conv2d" or inner.attrs.get("activation") is not None:
      raise NotImplementedError("relu must directly follow a linear conv2d layer")
    inner.attrs["activation"] = "relu"
    conv = inner
  if conv.op != "conv2d":
    raise NotImplementedError("max_pooling2d must follow conv2d (+relu) in a conv-stem subnetwork (got op %r)" % conv.op)
  if conv.attrs.get("activation") != "relu":
    raise NotImplementedError("the conv stem's activation must be relu")
  images = conv.inputs[0]
  if images.op != "placeholder" or len(images.shape) != 4:
    raise NotImplementedError("the conv stem must read the NHWC image feature directly")
  return conv, images


def _previous_members(previous_ensemble):
  """(iteration, name) of the previous ensemble's members, or None when it does not name them (MeanEnsemble): the
  iteration plan then checks the references against its frozen members."""
  wsubs = getattr(previous_ensemble, "weighted_subnetworks", None) if previous_ensemble is not None else None
  if previous_ensemble is not None and wsubs is None:
    return None
  return {(int(w.iteration_number), w.name) for w in (wsubs or [])}


def lower_subnetwork(builder, sub: subnetwork_lib.Subnetwork, variables: List[graph.Variable], train_op,
                     in_dim: int, logits_dim: int, iteration: int = 0, members=None) -> eng.SubnetworkPlanSpec:
  """`members`: the (iteration, name) of the previous ensemble's members, whose hidden layers the subnetwork may read
  through graph.concat (None: any stamped layer; the iteration plan checks it against its frozen members)."""
  if isinstance(sub.logits, dict):
    raise NotImplementedError("multi-head subnetworks are not implemented by the B200 engine")
  chain, inp, pieces = _trace_dense_chain(sub.logits, members, builder.name)
  if not chain:
    raise ValueError("subnetwork %s has no dense layer" % builder.name)
  if chain[-1].attrs.get("activation") is not None:
    raise NotImplementedError("the logits layer must be linear")
  for d in chain[:-1]:
    if d.attrs.get("activation") != "relu":
      raise NotImplementedError("hidden layers must use relu")
  if chain[-1].attrs.get("dropout_after") is not None:
    raise NotImplementedError("dropout on the logits is not implemented by the B200 engine")
  stem, image_shape = None, None
  if inp.op == "flatten":
    stem, images = _trace_conv_stem(inp)
    image_shape = tuple(int(v) for v in images.shape[1:])
    if int(np.prod(image_shape)) != in_dim:
      raise ValueError("subnetwork %s consumes images of shape %s, the input_fn provides %d values per example" % (
          builder.name, image_shape, in_dim))
  elif inp.shape[-1] != in_dim or len(inp.shape) != 2:
    raise ValueError("subnetwork %s consumes %s input features, the input_fn provides %d" % (builder.name, inp.shape[-1], in_dim))
  dims = [int(inp.shape[-1])] + [d.shape[-1] for d in chain]
  for ps in pieces:
    for p in ps or ():
      if p["src"] == "input" and (stem is not None or p["rows"][1] - p["rows"][0] != in_dim):
        raise NotImplementedError("subnetwork %s reads the input features as a piece of a concat that does not match "
                                  "them (%d values, conv stem: %s)" % (builder.name, in_dim, stem is not None))
  if dims[-1] != logits_dim:
    raise ValueError("subnetwork %s produces logits of dimension %d, head expects %d" % (builder.name, dims[-1], logits_dim))
  # last_layer must be the tensor feeding the logits layer (or the logits themselves)
  ll = sub.last_layer
  if ll is not chain[-1].inputs[0] and ll is not sub.logits:
    if not (isinstance(ll, graph.Tensor) and ll.op in ("relu", "dropout") and ll.inputs[0] is chain[-1].inputs[0]):
      raise NotImplementedError("last_layer must be the input of the logits layer (or the logits)")
  layers = ([stem] if stem is not None else []) + chain     # a conv stem's HWIO kernel / bias lead the lists
  ws = [np.array(d.attrs["kernel"].value, dtype=np.float32) for d in layers]
  bs = [np.array(d.attrs["bias"].value, dtype=np.float32) if d.attrs["bias"] is not None
        else np.zeros((d.shape[-1],), dtype=np.float32) for d in layers]
  if stem is not None and stem.attrs["bias"] is None:
    raise NotImplementedError("a conv stem without bias is not implemented")
  # train op: TrainOp from optimizer.minimize, or a TrainOpSpec wrapping one
  op = train_op.train_op if isinstance(train_op, subnetwork_lib.TrainOpSpec) else train_op
  if not isinstance(op, train.TrainOp):
    raise ValueError("build_subnetwork_train_op must return optimizer.minimize(...) / TrainOpSpec, got %r" % (op,))
  if op.kind == "no_op":
    opt_spec = ("sgd", 0.0)     # a frozen subnetwork (e.g. estimator_test.py _FrozenLinearBuilder)
  else:
    opt_spec = op.spec
    chain_vars = {id(d.attrs["kernel"]) for d in layers} | {id(d.attrs["bias"]) for d in layers if d.attrs["bias"] is not None}
    if op.var_list is not None and {id(v) for v in op.var_list} != chain_vars:
      raise NotImplementedError("training a strict subset of a subnetwork's variables is not implemented")
  complexity = float(np.asarray(sub.complexity, dtype=np.float32))
  spec = eng.SubnetworkPlanSpec(builder.name, dims, complexity, opt_spec, ws, bs, shared=sub.shared, image_shape=image_shape)
  # which tensor MATRIX mixture weights multiply (weighted.py:449): the logits themselves for sub-estimator builders
  # (autoensemble/common.py:115-118), the penultimate activation for simple_dnn-style builders
  spec.last_layer_is_logits = ll is sub.logits and len(chain) >= 1 and ll is not chain[-1].inputs[0]
  drops = [d.attrs.get("dropout_after") for d in chain[:-1]]
  spec.dropout = drops if any(v is not None for v in drops) else None
  spec.inputs = pieces if any(p is not None for p in pieces) else None
  for j, d in enumerate(chain):
    d.attrs[_LAYER] = (int(iteration), builder.name, j, j == len(chain) - 1)
  return spec


def build_and_lower(builder, feature_placeholders: Dict[str, graph.Tensor], labels_placeholder, head,
                    iteration_step, previous_ensemble, in_dim: int, config=None, iteration: int = 0):
  """One `_SubnetworkManager.build_subnetwork_spec` (ensemble_builder.py:679-805) against the symbolic graph, for
  AdaNet iteration `iteration` (what names the subnetwork's layers to later iterations)."""
  summary = _NullSummary()
  with graph.graph_scope() as g:
    sub = call_build_subnetwork(builder, feature_placeholders, labels_placeholder, head.logits_dimension, True,
                                iteration_step, summary, previous_ensemble, config)
    if not isinstance(sub, subnetwork_lib.Subnetwork):
      raise ValueError("build_subnetwork of %s must return an adanet Subnetwork" % builder.name)
    variables = list(g.variables)
    loss = head.create_loss(sub.logits)
    train_op = builder.build_subnetwork_train_op(subnetwork=sub, loss=loss, var_list=variables,
                                                 labels=labels_placeholder, iteration_step=iteration_step,
                                                 summary=summary, previous_ensemble=previous_ensemble)
  spec = lower_subnetwork(builder, sub, variables, train_op, in_dim, head.logits_dimension, iteration,
                          _previous_members(previous_ensemble))
  # bagging: a builder from an AutoEnsembleSubestimator with its own train_input_fn (autoensemble/common.py:151-180)
  spec.own_input = getattr(builder, "bagging_train_input_fn", None) is not None
  return spec, sub


# ---------------------------------------------------------------------------
# Tensors in Subnetwork.shared / persisted_tensors across checkpoints
# ---------------------------------------------------------------------------

_REF_TAG = "__adanet_layer__"


def _tensor_ref(t: graph.Tensor):
  """[iteration, name, layer] of a lowered subnetwork's layer, or "input" for the input features."""
  while t.op in ("relu", "dropout"):
    t = t.inputs[0]
  if t.op == "member_layer":
    return list(t.attrs["ref"])
  if t.op == "dense" and _LAYER in t.attrs:
    return list(t.attrs[_LAYER][:3])
  if t.op in ("input_layer", "input_ref"):
    return "input"
  raise ValueError("a tensor produced by op %r cannot be saved in a checkpoint: only subnetwork layers, the input "
                   "features and concats of them can" % t.op)


def encode_tensors(obj):
  """`obj` (a Subnetwork's shared / persisted_tensors value) with every graph Tensor replaced by a tagged reference:
  {"__adanet_layer__": [iteration, name, layer]} for a layer, {"__adanet_layer__": [[...], ...]} for a concat of them
  (nested concats flattened).  Everything else is returned as is."""
  if isinstance(obj, graph.Tensor):
    if obj.op == "concat" or (obj.op == "relu" and obj.inputs[0].op == "concat"):
      elems = []
      _flatten_concat(obj, False, elems)
      return {_REF_TAG: [_tensor_ref(e) for e, _ in elems]}
    return {_REF_TAG: _tensor_ref(obj)}
  if isinstance(obj, dict):
    out = {k: encode_tensors(v) for k, v in obj.items()}
    return obj if all(out[k] is obj[k] for k in obj) else out
  if isinstance(obj, (list, tuple)):
    out = [encode_tensors(v) for v in obj]
    return obj if all(a is b for a, b in zip(out, obj)) else type(obj)(out)
  return obj


def layer_handle(ref, dims_of, in_dim: int) -> graph.Tensor:
  """The graph handle of one reference: lowers to that member's layer (or to the input features for "input").
  `dims_of(iteration, name)`: the member's dims."""
  if ref == "input":
    return graph.Tensor((None, in_dim), "input_ref")
  it, name, j = int(ref[0]), ref[1], int(ref[2])
  dims = dims_of(it, name)
  return graph.Tensor((None, int(dims[j + 1])), "member_layer", (), {"ref": (it, name, j), "is_logits": j == len(dims) - 2})


def decode_tensors(obj, dims_of, in_dim: int):
  """Inverse of encode_tensors: tagged references become graph handles (a concat of handles for a list)."""
  if isinstance(obj, dict):
    if set(obj) == {_REF_TAG}:
      ref = obj[_REF_TAG]
      if isinstance(ref, list) and ref and isinstance(ref[0], (list, str)):
        return graph.concat([layer_handle(r, dims_of, in_dim) for r in ref])
      return layer_handle(ref, dims_of, in_dim)
    return {k: decode_tensors(v, dims_of, in_dim) for k, v in obj.items()}
  if isinstance(obj, list):
    return [decode_tensors(v, dims_of, in_dim) for v in obj]
  return obj


def member_last_layer(iteration: int, name: str, dims, inputs, dims_of, in_dim: int) -> graph.Tensor:
  """A restored member's Subnetwork.last_layer: the input of its logits layer as handles (its pieces' concat)."""
  n = len(dims) - 1
  own = [iteration, name, n - 2] if n >= 2 else "input"
  ps = inputs[-1] if inputs else None
  if not ps:
    return layer_handle(own, dims_of, in_dim)
  refs = [own if p["src"] == "own" else ("input" if p["src"] == "input" else [p["iteration"], p["name"], p["layer"]])
          for p in ps]
  return graph.concat([layer_handle(r, dims_of, in_dim) for r in refs])


def restored_subnetwork(member: dict, dims_of, in_dim: int) -> subnetwork_lib.Subnetwork:
  """The Subnetwork a later iteration's builders see for a member restored from its ensemble-latest.json record: its
  logits, last_layer and the tensors of shared / persisted_tensors as handles that lower to the same layers as the
  live member's tensors (its logits are refused as a concat piece, as the live ones are)."""
  it, name, dims = int(member["iteration"]), member["name"], member["dims"]
  return subnetwork_lib.Subnetwork(
      last_layer=member_last_layer(it, name, dims, member.get("inputs"), dims_of, in_dim),
      logits=layer_handle([it, name, len(dims) - 2], dims_of, in_dim), complexity=member["complexity"],
      shared=decode_tensors(member["shared"], dims_of, in_dim),
      persisted_tensors=decode_tensors(member.get("persisted_tensors"), dims_of, in_dim))
