"""Subnetworks that read the hidden layers of previous-iteration subnetworks through graph.concat, on the host:
concat shapes and errors, the pieces each accepted pattern lowers to, the refusals, tagged references of tensors in
`shared` through JSON, and the fp64 reference's connected forward / backward against the materialised concat."""

import json

import numpy as np
import pytest

import adanet_b200 as adanet
from adanet_b200 import graph
from adanet_b200 import heads
from adanet_b200 import train
from adanet_b200.core import engine as eng
from adanet_b200.core import lowering
from tests import connected_oracle as co

IN = 6
C = 3


class Example(adanet.subnetwork.Builder):
  """The issue's example builder: one hidden layer, the previous member's exposed `hidden` concatenated onto it."""

  def __init__(self, name="ex", width=8, key="shared", seed=0):
    self._name, self._width, self._key, self._seed = name, width, key, seed

  @property
  def name(self):
    return self._name

  def _hidden(self, prev):
    sub = prev.weighted_subnetworks[-1].subnetwork
    return sub.shared["hidden"] if self._key == "shared" else (
        sub.persisted_tensors["hidden_layer"] if self._key == "persisted" else sub.last_layer)

  def build_subnetwork(self, features, logits_dimension, training, iteration_step, summary, previous_ensemble=None):
    x = graph.input_layer(features, [graph.numeric_column("x", IN)])
    h = graph.dense(x, self._width, activation=graph.relu, kernel_initializer=graph.glorot_uniform_initializer(self._seed))
    if previous_ensemble:
      h = graph.concat([h, self._hidden(previous_ensemble)], axis=-1)
    logits = graph.dense(h, logits_dimension, kernel_initializer=graph.glorot_uniform_initializer(self._seed + 1))
    return adanet.Subnetwork(last_layer=h, logits=logits, complexity=1.0, shared={"hidden": h},
                             persisted_tensors={"hidden_layer": h})

  def build_subnetwork_train_op(self, subnetwork, loss, var_list, labels, iteration_step, summary, previous_ensemble):
    return train.GradientDescentOptimizer(0.1).minimize(loss, var_list)


class Fn(Example):
  """A builder whose graph is `fn(x, prev_sub, logits_dimension) -> (last_layer, logits)`."""

  def __init__(self, fn, name="fn"):
    super().__init__(name)
    self._fn = fn

  def build_subnetwork(self, features, logits_dimension, training, iteration_step, summary, previous_ensemble=None):
    x = graph.input_layer(features, [graph.numeric_column("x", IN)])
    prev = previous_ensemble.weighted_subnetworks[-1].subnetwork if previous_ensemble else None
    ll, logits = self._fn(x, prev, logits_dimension)
    return adanet.Subnetwork(last_layer=ll, logits=logits, complexity=1.0, shared={"hidden": ll})


def _lower(builder, prev=None, it=0):
  ph = {"x": graph.placeholder(IN, "x")}
  return lowering.build_and_lower(builder, ph, None, heads.MultiClassHead(C), 0, prev, in_dim=IN, iteration=it)


def _ens(members):
  """previous_ensemble over [(iteration, name, Subnetwork)]."""
  ws = [adanet.WeightedSubnetwork(name=n, iteration_number=t, subnetwork=s) for t, n, s in members]
  return adanet.ComplexityRegularized(ws, bias=0, logits=None)


def _mem(it, name, layer, r0, r1):
  return {"src": "member", "iteration": it, "name": name, "layer": layer, "rows": [r0, r1]}


def test_concat_shapes_and_errors():
  a, b = graph.placeholder(3, "a"), graph.placeholder(5, "b")
  c = graph.concat([a, b], axis=-1)
  assert c.shape == (None, 8) and c.op == "concat" and c.inputs == (a, b)
  assert graph.concat([a, b], axis=1).shape == (None, 8)
  assert graph.concat([graph.concat([a, b]), a]).shape == (None, 11)
  with pytest.raises(NotImplementedError, match="last axis"):
    graph.concat([a, b], axis=0)
  img = graph.placeholder((4, 4, 2), "img")
  with pytest.raises(NotImplementedError, match="rank-2"):
    graph.concat([img, img])
  with pytest.raises(ValueError, match="different ranks"):
    graph.concat([a, img])
  with pytest.raises(ValueError, match="out of range"):
    graph.concat([a, b], axis=2)
  with pytest.raises(ValueError, match="batch"):
    graph.concat([graph.Tensor((4, 3), "placeholder"), graph.Tensor((5, 3), "placeholder")])
  with pytest.raises(ValueError):
    graph.concat([])


def test_example_builder_over_four_iterations_then_the_piece_limit():
  """The example builder grows its logits layer's pieces by one per iteration: 2, 3, 4 pieces, then 5 raises."""
  members, widths = [], [8, 5, 7, 6, 4]
  spec0, sub0 = _lower(Example("b0", widths[0]), None, 0)
  assert spec0.inputs is None and spec0.dims == [IN, 8, C]
  members.append((0, "b0", sub0))
  for t in range(1, 4):
    spec, sub = _lower(Example("b%d" % t, widths[t]), _ens(members), t)
    want = [{"src": "own", "rows": [0, widths[t]]}]
    r = widths[t]
    for k in range(t - 1, -1, -1):          # the previous member's exposure: its own layer, then what it read
      want.append(_mem(k, "b%d" % k, 0, r, r + widths[k]))
      r += widths[k]
    assert spec.inputs == [None, want]
    assert spec.dims == [IN, widths[t], C] and spec.ws[1].shape == (r, C)
    members.append((t, "b%d" % t, sub))
  with pytest.raises(NotImplementedError, match="at most 4"):
    _lower(Example("b4", widths[4]), _ens(members), 4)


@pytest.mark.parametrize("key", ["persisted", "last_layer"])
def test_persisted_tensors_and_last_layer_resolve_like_shared(key):
  _, sub0 = _lower(Example("b0", 8), None, 0)
  spec, _ = _lower(Example("b1", 5, key=key), _ens([(0, "b0", sub0)]), 1)
  assert spec.inputs == [None, [{"src": "own", "rows": [0, 5]}, _mem(0, "b0", 0, 5, 13)]]


def _two_layer_member():
  def fn(x, prev, C_):
    h0 = graph.dense(x, 4, activation=graph.relu)
    h1 = graph.dense(h0, 7, activation=graph.relu)
    return h1, graph.dense(h1, C_)
  _, sub = _lower(Fn(fn, "m"), None, 0)
  return sub


def test_accepted_patterns_lower_to_pieces_and_rows():
  m = _two_layer_member()
  prev = _ens([(0, "m", m)])
  h0_m = m.logits.inputs[0].inputs[0]          # the member's layer 0 (its layer 1 is m.last_layer)

  # the reference's pattern with relu for leaky_relu: relu(concat([dense(x, use_bias=False), prev_hidden]))
  def ref_pattern(x, p, C_):
    h = graph.relu(graph.concat([graph.dense(x, 10, use_bias=False), p.last_layer]))
    return h, graph.dense(h, C_)
  spec, _ = _lower(Fn(ref_pattern), prev, 1)
  assert spec.inputs == [None, [{"src": "own", "rows": [0, 10]}, _mem(0, "m", 1, 10, 17)]]
  assert spec.dims == [IN, 10, C] and not spec.bs[0].any()

  # nested concats flatten; a dropout / relu wrapper around a member layer names that layer; the member read first
  def nested(x, p, C_):
    h = graph.dense(x, 9, activation=graph.relu)
    cat = graph.concat([graph.concat([graph.dropout(p.last_layer, 0.5, training=True), h]), graph.relu(h0_m)])
    return cat, graph.dense(cat, C_)
  spec, _ = _lower(Fn(nested), prev, 1)
  assert spec.inputs == [None, [_mem(0, "m", 1, 0, 7), {"src": "own", "rows": [7, 16]}, _mem(0, "m", 0, 16, 20)]]

  # the first layer reads a member's layer 1 next to the input features; its own dropout stays its own
  def first(x, p, C_):
    h = graph.dropout(graph.dense(graph.concat([x, p.last_layer]), 12, activation=graph.relu), 0.25, seed=5, training=True)
    h2 = graph.dense(graph.concat([h, h0_m, x]), 6, activation=graph.relu)
    return h2, graph.dense(h2, C_)
  spec, _ = _lower(Fn(first), prev, 1)
  assert spec.inputs == [[{"src": "own", "rows": [0, IN]}, _mem(0, "m", 1, IN, IN + 7)],
                         [{"src": "own", "rows": [0, 12]}, _mem(0, "m", 0, 12, 16), {"src": "input", "rows": [16, 16 + IN]}],
                         None]
  assert spec.dims == [IN, 12, 6, C] and spec.dropout == [(0.25, 5), None]
  assert [w.shape for w in spec.ws] == [(IN + 7, 12), (12 + 4 + IN, 6), (6, C)]

  # a member's exposed concat expands into that member's own pieces
  def expose(x, p, C_):
    h = graph.dense(x, 3, activation=graph.relu)
    cat = graph.concat([h, p.last_layer])
    return cat, graph.dense(cat, C_)
  _, sub1 = _lower(Fn(expose, "e"), prev, 1)
  spec, _ = _lower(Fn(lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(
      graph.concat([graph.dense(x, 2, activation=graph.relu), p.shared["hidden"]])), "f"),
      _ens([(0, "m", m), (1, "e", sub1)]), 2)
  assert spec.inputs == [None, [{"src": "own", "rows": [0, 2]}, _mem(1, "e", 0, 2, 5), _mem(0, "m", 1, 5, 12)]]
  # a plain chain keeps inputs None
  spec, _ = _lower(Example("plain", 4), None, 0)
  assert spec.inputs is None


def test_lowering_refusals():
  m = _two_layer_member()
  prev = _ens([(0, "m", m)])
  cases = [
      # a skip connection inside one subnetwork
      (lambda x, p, C_: (lambda h0: (lambda h1: (graph.concat([h1, h0]), graph.dense(graph.concat([h1, h0]), C_)))(
          graph.dense(h0, 4, activation=graph.relu)))(graph.dense(x, 4, activation=graph.relu)), "skip connection"),
      # a layer that reads only another subnetwork's layers
      (lambda x, p, C_: (p.last_layer, graph.dense(graph.concat([p.last_layer]), C_)), "reads only hidden layers"),
      (lambda x, p, C_: (p.last_layer, graph.dense(p.last_layer, C_)), "directly"),
      # a member's logits
      (lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(graph.concat([graph.dense(x, 4, activation=graph.relu),
                                                                           p.logits])), "logits"),
      # relu(concat) over the input features
      (lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(graph.relu(graph.concat([x, p.last_layer]))), "input features"),
      # more pieces than the kernel runs
      (lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(graph.concat(
          [graph.dense(x, 4, activation=graph.relu)] + [p.last_layer] * 4)), "at most 4"),
  ]
  for fn, msg in cases:
    with pytest.raises(NotImplementedError, match=msg):
      _lower(Fn(fn), prev, 1)
  # a layer of a subnetwork that is not in the previous ensemble
  with pytest.raises(NotImplementedError, match="not a member"):
    _lower(Example("x"), _ens([(3, "other", m)]), 4)


def test_conv_stem_output_and_images_cannot_be_pieces():
  class Stem(Example):
    def build_subnetwork(self, features, logits_dimension, training, iteration_step, summary, previous_ensemble=None):
      img = features["img"]
      flat = graph.flatten(graph.max_pooling2d(graph.conv2d(img, 2, 3, padding="same", activation=graph.relu)))
      h = graph.dense(flat, 4, activation=graph.relu)
      other = graph.flatten(graph.max_pooling2d(graph.conv2d(img, 2, 3, padding="same", activation=graph.relu)))
      cat = graph.concat([h, other])
      return adanet.Subnetwork(last_layer=cat, logits=graph.dense(cat, logits_dimension), complexity=1.0)

  ph = {"img": graph.placeholder((4, 4, 1), "img")}
  with pytest.raises(NotImplementedError, match="conv-stem output"):
    lowering.build_and_lower(Stem(), ph, None, heads.MultiClassHead(C), 0, None, in_dim=16)


def _net_stub(name, it, dims, inputs=None):
  class N:
    pass
  n = N()
  n.name, n.iteration, n.dims, n.inputs = name, it, dims, inputs
  return n


def test_plan_refusals_raise_before_anything_runs(monkeypatch):
  """IterationPlan's host-side checks (_check_connected) for connected candidates: SIMT path, row-sharded, bagged,
  MATRIX over a concatenated last_layer, and a member that is not frozen.  They run before any allocation."""
  member = _net_stub("m", 0, [IN, 4, C])
  spec = eng.SubnetworkPlanSpec("c", [IN, 5, C], 1.0, ("sgd", 0.1), [np.zeros((IN, 5)), np.zeros((9, C))],
                                [np.zeros(5), np.zeros(C)], inputs=[None, [{"src": "own", "rows": [0, 5]},
                                                                           _mem(0, "m", 0, 5, 9)]])
  ens = eng.EnsemblerPlanSpec()
  monkeypatch.setattr(eng, "planes_enabled", lambda: True)
  eng._check_connected([spec], [0], [member], ens, None, {})           # accepted
  with pytest.raises(NotImplementedError, match="row-sharded"):
    eng._check_connected([spec], [0], [member], ens, None, {0: object()})
  with pytest.raises(NotImplementedError, match="bagged"):
    from dataclasses import replace
    eng._check_connected([replace(spec, own_input=True)], [0], [member], ens, None, {})
  with pytest.raises(NotImplementedError, match="MATRIX"):
    eng._check_connected([spec], [0], [member], eng.EnsemblerPlanSpec(mixture_weight_type="matrix"), None, {})
  with pytest.raises(NotImplementedError, match="MATRIX"):
    eng._check_connected([], [], [member, _net_stub("c", 1, spec.dims, spec.inputs)],
                         eng.EnsemblerPlanSpec(mixture_weight_type="matrix"), None, {})
  with pytest.raises(NotImplementedError, match="not a frozen member"):
    eng._check_connected([spec], [0], [], ens, None, {})
  monkeypatch.setattr(eng, "planes_enabled", lambda: False)
  with pytest.raises(NotImplementedError, match="plane path"):
    eng._check_connected([spec], [0], [member], ens, None, {})


def test_search_refuses_candidates_that_drop_a_member_they_read():
  from adanet_b200.core import search as srch
  s = srch.AdaNetSearch.__new__(srch.AdaNetSearch)
  s.frozen = [_net_stub("a", 0, [IN, 4, C]), _net_stub("b", 1, [IN, 4, C], [None, [{"src": "own", "rows": [0, 4]},
                                                                                    _mem(0, "a", 0, 4, 8)]])]
  spec = eng.SubnetworkPlanSpec("c", [IN, 5, C], 1.0, ("sgd", 0.1), [], [],
                                inputs=[None, [{"src": "own", "rows": [0, 5]}, _mem(1, "b", 0, 5, 9)]])
  plain = eng.SubnetworkPlanSpec("p", [IN, C], 1.0, ("sgd", 0.1), [], [])
  s._check_kept_members([spec, plain], srch.strategy_candidates(["grow", "solo"], ["c", "p"])[:2] +
                        [srch.EnsembleCandidate("p_solo", [1], False)])
  with pytest.raises(NotImplementedError, match="c_solo drops b"):
    s._check_kept_members([spec, plain], srch.strategy_candidates(["solo"], ["c", "p"]))
  # a kept member that reads a dropped one
  with pytest.raises(NotImplementedError, match="drops a .* b reads"):
    s._check_kept_members([spec, plain], [srch.EnsembleCandidate("prune", [1], [1])])


def test_shared_tensors_round_trip_through_json():
  _, sub0 = _lower(Example("b0", 8), None, 0)
  _, sub1 = _lower(Example("b1", 5), _ens([(0, "b0", sub0)]), 1)
  shared = {"hidden": sub1.shared["hidden"], "n": 3, "nested": {"h0": sub0.shared["hidden"], "xs": [1.5, "a"]}}
  enc = lowering.encode_tensors(shared)
  assert enc == {"hidden": {"__adanet_layer__": [[1, "b1", 0], [0, "b0", 0]]}, "n": 3,
                 "nested": {"h0": {"__adanet_layer__": [0, "b0", 0]}, "xs": [1.5, "a"]}}
  plain = {"num_layers": 2, "x": [1, 2]}
  assert lowering.encode_tensors(plain) is plain and lowering.encode_tensors(None) is None
  dims = {(0, "b0"): [IN, 8, C], (1, "b1"): [IN, 5, C]}
  back = lowering.decode_tensors(json.loads(json.dumps(enc)), lambda it, n: dims[(it, n)], IN)
  assert back["n"] == 3 and back["nested"]["xs"] == [1.5, "a"]
  assert back["hidden"].op == "concat" and back["hidden"].shape == (None, 13)
  assert back["nested"]["h0"].op == "member_layer" and back["nested"]["h0"].attrs["ref"] == (0, "b0", 0)
  assert lowering.encode_tensors(back) == enc
  # restored handles lower to the same member layers as the live tensors
  restored = adanet.Subnetwork(last_layer=back["hidden"], logits=graph.placeholder(C, "l"), complexity=1.0, shared=back)
  live, _ = _lower(Example("b2", 4), _ens([(0, "b0", sub0), (1, "b1", sub1)]), 2)
  again, _ = _lower(Example("b2", 4), _ens([(0, "b0", sub0), (1, "b1", restored)]), 2)
  assert live.inputs == again.inputs
  ll = lowering.member_last_layer(1, "b1", [IN, 5, C], live.inputs and [None, [{"src": "own", "rows": [0, 5]},
                                                                             _mem(0, "b0", 0, 5, 13)]],
                                  lambda it, n: dims[(it, n)], IN)
  assert lowering.encode_tensors(ll) == enc["hidden"]
  # a restored member's logits cannot be a piece
  lg = lowering.layer_handle([0, "b0", 1], lambda it, n: dims[(it, n)], IN)
  with pytest.raises(NotImplementedError, match="logits"):
    _lower(Fn(lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(graph.concat([graph.dense(x, 2), lg]))),
           _ens([(0, "b0", sub0)]), 1)


def test_oracle_connected_forward_backward_equal_the_materialised_concat():
  rng = np.random.default_rng(7)
  B = 33
  x = rng.standard_normal((B, IN))
  mws = [rng.standard_normal((IN, 40)), rng.standard_normal((40, 100)), rng.standard_normal((100, C))]
  mbs = [rng.standard_normal(40), rng.standard_normal(100), rng.standard_normal(C)]
  member_acts = {(0, "m"): co.connected_forward(mws, mbs, x, None, {})[0]}
  inputs = [[{"src": "own", "rows": [0, IN]}, _mem(0, "m", 1, IN, IN + 100)],
            [_mem(0, "m", 0, 0, 40), {"src": "own", "rows": [40, 104]}, {"src": "input", "rows": [104, 104 + IN]}],
            None]
  ws = [rng.standard_normal((IN + 100, 64)) * 0.1, rng.standard_normal((104 + IN, 30)) * 0.1, rng.standard_normal((30, C))]
  bs = [rng.standard_normal(64), rng.standard_normal(30), rng.standard_normal(C)]
  drop = ([(0.3, 11), None], 4)
  acts, xs = co.connected_forward(ws, bs, x, inputs, member_acts, drop)
  # materialised: concat the pieces, one GEMM per layer
  ma = member_acts[(0, "m")]
  cat0 = np.concatenate([x, ma[2]], axis=1)
  h0 = np.maximum(cat0 @ ws[0] + bs[0], 0)
  from oracle import adanet_oracle as orc
  keep = orc.dropout_keep_mask(11, 0, 4, B, 64, 0.3)
  h0 = np.where(keep, h0 / 0.7, 0)
  cat1 = np.concatenate([ma[1], h0, x], axis=1)
  h1 = np.maximum(cat1 @ ws[1] + bs[1], 0)
  lg = h1 @ ws[2] + bs[2]
  for got, want in zip(acts[1:], [h0, h1, lg]):
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
  dl = rng.standard_normal((B, C))
  dws, dbs, dxs = co.connected_backward(ws, acts, xs, dl, inputs, drop)
  dz2 = dl
  dh1 = dz2 @ ws[2].T
  dz1 = dh1 * (h1 > 0)
  dcat1 = dz1 @ ws[1].T
  dh0 = dcat1[:, 40:104] / 0.7
  dz0 = dh0 * (h0 > 0)
  for got, want in zip(dws, [cat0.T @ dz0, cat1.T @ dz1, h1.T @ dz2]):
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
  for got, want in zip(dbs, [dz0.sum(0), dz1.sum(0), dz2.sum(0)]):
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
  np.testing.assert_allclose(dxs[1], dcat1[:, 40:104], rtol=1e-12, atol=1e-12)
  np.testing.assert_allclose(dxs[2], dh1, rtol=1e-12, atol=1e-12)


def test_restored_member_resolves_like_the_live_one():
  """A member restored from its ensemble-latest.json record: its shared / last_layer lower to the same pieces as the
  live member's, and its logits are refused as a piece (they are not mistaken for the input features, also when the
  logits have the input's width)."""
  _, sub0 = _lower(Example("b0", 8), None, 0)
  spec1, sub1 = _lower(Example("b1", 5), _ens([(0, "b0", sub0)]), 1)
  dims = {(0, "b0"): [IN, 8, IN], (1, "b1"): [IN, 5, IN]}         # logits as wide as the input features
  recs = [{"name": "b0", "iteration": 0, "complexity": 1.0, "dims": dims[(0, "b0")], "shared": lowering.encode_tensors(sub0.shared)},
          {"name": "b1", "iteration": 1, "complexity": 1.0, "dims": dims[(1, "b1")], "inputs": spec1.inputs,
           "shared": lowering.encode_tensors(sub1.shared),
           "persisted_tensors": lowering.encode_tensors(sub1.persisted_tensors)}]
  restored = [lowering.restored_subnetwork(r, lambda it, n: dims[(it, n)], IN) for r in recs]
  prev = _ens([(0, "b0", restored[0]), (1, "b1", restored[1])])
  live = _ens([(0, "b0", sub0), (1, "b1", sub1)])
  for key in ("shared", "persisted", "last_layer"):
    want, _ = _lower(Example("b2", 4, key=key), live, 2)
    got, _ = _lower(Example("b2", 4, key=key), prev, 2)
    assert got.inputs == want.inputs
  reads_logits = lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(graph.concat([graph.dense(x, 3), p.logits]))
  for ens in (live, prev):
    with pytest.raises(NotImplementedError, match="logits"):
      _lower(Fn(reads_logits), ens, 2)


def test_input_pieces_must_be_the_plain_input_layer():
  """The input features inside a concat: graph.input_layer only -- a raw placeholder could be anything (labels,
  another tensor of the same width), and dropout or relu on the input features is not implemented, as outside a
  concat."""
  m = _two_layer_member()
  prev = _ens([(0, "m", m)])
  cases = [
      (lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(graph.concat(
          [graph.dense(x, 4, activation=graph.relu), graph.dropout(x, 0.5, training=True), p.last_layer])), "dropout"),
      (lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(graph.concat(
          [graph.dense(x, 4, activation=graph.relu), graph.relu(x), p.last_layer])), "relu or dropout"),
      (lambda x, p, C_: (lambda c: (c, graph.dense(c, C_)))(graph.concat(
          [graph.dense(x, 4, activation=graph.relu), graph.placeholder(IN, "other"), p.last_layer])), "raw placeholder"),
  ]
  for fn, msg in cases:
    with pytest.raises(NotImplementedError, match=msg):
      _lower(Fn(fn), prev, 1)
