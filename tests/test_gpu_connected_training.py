"""Training subnetworks that read the hidden layers of previous-iteration subnetworks (graph.concat lowered to
SubnetworkPlanSpec.inputs), on the GPU:

  step      teacher-forced IterationPlan steps against float64 in both plane formats: candidates read frozen hidden
            layers at their first, hidden and logits layers, with piece widths on and off the k-block grid; one reads
            a frozen member's layer 1 from its own layer 0, one has dropout, and one frozen member itself reads
            another.  Each layer's output from the engine's own piece inputs, each piece's dW, dX (through db of the
            layer below), the update and each piece's weight planes are checked with the bounds of
            test_gpu_step_state
  search    three iterations of the example builder through Estimator.train under SCALAR and VECTOR mixture weights:
            winners and architecture equal the float64 reference's (tests/connected_oracle.py), per-step losses
            within 1e-5 (sub_loss, adanet_loss, EMA); evaluate / predict from a fresh Estimator on the model_dir match
            the reference; a kill at an iteration boundary and an in-flight resume (Momentum: per-piece slots) end
            identical to the uninterrupted run
  fallback  an fp16 overflow in an iteration whose frozen members include a connected one: the TF32 re-run matches
            the reference
  slots     per-piece Momentum slots through state_dict / load_state_dict: the next step is byte-identical
  ranks     two ranks on one GPU over gloo, the winners owned by rank 1: rank 0's replicas of connected members,
            their piece planes and the next iterations are identical on both ranks
"""

import json
import os

import numpy as np
import pytest

from tests import connected_oracle as co
from tests.parity_util import orc
from tests import test_gpu_step_state as st

D, C, B = 100, 10, 512


def _mem(it, name, layer, r0, r1):
  return {"src": "member", "iteration": it, "name": name, "layer": layer, "rows": [r0, r1]}


def _own(r0, r1):
  return {"src": "own", "rows": [r0, r1]}


def _glorot(rng, a, b):
  lim = np.sqrt(6.0 / (a + b))
  return rng.uniform(-lim, lim, size=(a, b)).astype(np.float32)


def _params(rng, dims, inputs):
  ws, bs = [], []
  for i in range(len(dims) - 1):
    rows = inputs[i][-1]["rows"][1] if inputs and inputs[i] else dims[i]
    ws.append(_glorot(rng, rows, dims[i + 1]))
    bs.append((rng.standard_normal(dims[i + 1]) * 0.05).astype(np.float32))
  return ws, bs


# frozen: m0 plain 100 -> 40 -> 130 -> C (widths on and off the k-block grid); m1 reads m0's layer 1 from its layer 0
FROZEN = [("m0", [D, 40, 130, C], None),
          ("m1", [D, 64, C], [[_own(0, D), _mem(0, "m0", 1, D, D + 130)], None])]
CANDS = [
    # the first layer reads a frozen member's layer 1 (a layer the forward computes one wave later)
    ("first", [D, 64, C], [[_own(0, D), _mem(0, "m0", 1, D, D + 130)], None], None),
    # a hidden layer reads two frozen layers (one of them a connected member's) and the input features
    ("hidden", [D, 100, 40, C], [None, [_mem(0, "m0", 0, 0, 40), _own(40, 140), _mem(1, "m1", 0, 140, 204),
                                        {"src": "input", "rows": [204, 304]}], None], [(0.25, 17), None]),
    # the logits layer reads the frozen last hidden layers (the example builder's shape)
    ("logits", [D, 130, C], [None, [_own(0, 130), _mem(1, "m1", 0, 130, 194), _mem(0, "m0", 1, 194, 324)]], None),
    ("plain", [D, 64, C], None, None),
]
LR = 0.05
ENS = dict(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001)


def _build(rng):
  import torch
  from adanet_b200.core import engine as eng
  dev = torch.device("cuda", torch.cuda.current_device())
  fnets, fparams = [], []
  for k, (name, dims, inputs) in enumerate(FROZEN):
    ws, bs = _params(rng, dims, inputs)
    fparams.append((ws, bs))
    fnets.append(eng.DenseNet(name, dims, ws, bs, 1.0 + k, B, dev, iteration=k, inputs=inputs, members=list(fnets)))
  specs, cparams = [], []
  for name, dims, inputs, drop in CANDS:
    ws, bs = _params(rng, dims, inputs)
    cparams.append((ws, bs))
    specs.append(eng.SubnetworkPlanSpec(name, dims, 2.0, ("sgd", LR), [w.copy() for w in ws], [b.copy() for b in bs],
                                        dropout=drop, inputs=inputs))
  plan = eng.IterationPlan(2, specs, fnets, eng.EnsemblerPlanSpec(**ENS), B, D, C, "softmax_xent", device=dev)
  return plan, fnets, fparams


def _piece_input(net, i, k, x, frozen_acts, acts):
  p = net.pieces(i)[k]
  if p["src"] == "own":
    return acts[i]
  if p["src"] == "input":
    return st.f64(x)
  return frozen_acts[(p["iteration"], p["name"])][p["layer"] + 1]


def _check_step(fails, plan, fnets, pre, post, x, y, step_dev, f16):
  floor_x = st.F16_FLOOR if f16 else 0.0
  # frozen members: each layer from the engine's own piece inputs
  frozen_acts = {}
  for f in fnets:
    acts = [st.f64(x)] + st._acts(f, B, True)
    n = len(f.ws)
    for i in range(n):
      h = np.concatenate([_piece_input(f, i, k, x, frozen_acts, acts) for k in range(len(f.pieces(i)))], axis=1)
      exact, bound = st.layer_fwd(h, f.ws[i].cpu().numpy(), f.bs[i].cpu().numpy(), i < n - 1, floor=floor_x)
      got = f.logits.cpu().numpy() if i == n - 1 else acts[i + 1]
      st._check(fails, "forward", got, exact, bound, "frozen %s layer %d" % (f.name, i))
    frozen_acts[(f.iteration, f.name)] = acts + [f.logits.cpu().numpy()]
  for c, (name, dims, inputs, drop) in zip(plan.candidates, CANDS):
    key, n, net = "c%d_" % c.index, len(c.net.ws), c.net
    acts = [st.f64(x)] + st._acts(net, B, True)
    logits = net.logits.cpu().numpy()
    hs, masks, muls = [], [None], [1.0]
    for i in range(n):
      h = np.concatenate([_piece_input(net, i, k, x, frozen_acts, acts) for k in range(len(net.pieces(i)))], axis=1)
      hs.append(h)
      w, b = pre[key + "w%d" % i], pre[key + "b%d" % i]
      d = drop[i] if (drop and i < n - 1) else None
      keep = orc.dropout_keep_mask(d[1], i, step_dev, B, w.shape[1], d[0]) if d else None
      exact, bound = st.layer_fwd(h, w, b, i < n - 1, keep, float(np.float32(d[0])) if d else 0.0, floor_x)
      got = logits if i == n - 1 else acts[i + 1]
      st._check(fails, "forward", got, exact, bound, "%s layer %d" % (name, i))
      if i < n - 1:
        st._plane_checks(fails, net.hp[i], B, w.shape[1], got, "%s layer %d" % (name, i))
        masks.append(got > 0)
        muls.append(st._dx_mul(d))
    dl = st.check_heads(fails, {"head": "softmax_xent"}, c, logits, y, name)
    # dW from the concatenated piece inputs; dX only through the primary piece's rows
    wdx = [pre[key + "w%d" % i][slice(*net.piece_rows(i)[net.primary(i)])] for i in range(n)]
    floor_g = st.F16_FLOOR * 2.0 ** -c.dz_log2 if f16 else 0.0
    bw = st.backward(wdx, hs, dl, masks, muls, floor_g, floor_x)
    grads = []
    for i in range(n):
      dw = (np.concatenate([t.cpu().numpy() for t in c.piece_dws[i]], axis=0) if c.piece_dws[i] is not None
            else c.dws[i].cpu().numpy())
      st._check(fails, "backward", dw, bw["dw"][i], bw["dw_b"][i], "%s dW%d (%d pieces)" % (name, i, len(net.pieces(i))))
      if i < n - 1:
        st._check(fails, "backward", c.dbs[i].cpu().numpy(), bw["db"][i], bw["db_b"][i], "%s db%d" % (name, i))
      grads += [dw, c.dbs[i].cpu().numpy()]
    names = [key + nm for i in range(n) for nm in ("w%d" % i, "b%d" % i)]
    st.check_update(fails, ("sgd", LR), [pre[nm] for nm in names], grads, pre, post, key + "sub_opt_", names, name)
    st.check_planes_resplit(fails, [("W%d piece %d" % (i, k), net.ws[i][r0:r1], wp) for i in range(n)
                                    for k, ((r0, r1), wp) in enumerate(zip(net.piece_rows(i), net.piece_wps[i]))], name)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt_name", ["f16", "tf32"])
def test_connected_steps_match_fp64(fmt_name):
  import torch
  from adanet_b200 import _lib
  from tests.test_gpu_plane_groups import _open, _set_format
  _open()
  before = _lib.plane_format()
  _set_format(_lib, fmt_name)
  _lib.plane_overflow()
  try:
    rng = np.random.default_rng(11)
    plan, fnets, _ = _build(rng)
    # the frozen member layer the "first" candidate reads is one wave later: its layer 0 runs at level 2
    lv = __import__("adanet_b200.core.engine", fromlist=["_levels"])._levels(list(fnets) + [c.net for c in plan.candidates])
    assert lv[(id(plan.candidates[0].net), 0)] == 2 and lv[(id(fnets[1]), 0)] == 2
    x, y = orc.make_tabular(B * 3, D, C, seed=5)
    fails = []
    for k in range(3):
      pre = plan.state_dict()
      xb, yb = x[k * B:(k + 1) * B], y[k * B:(k + 1) * B]
      plan.train_step(xb, yb)
      torch.cuda.synchronize()
      post = plan.state_dict()
      _check_step(fails, plan, fnets, pre, post, xb, yb, int(pre["step_dev"]), fmt_name == "f16")
    # state_dict round-trips the per-piece optimizer state and weights
    st2 = plan.state_dict()
    plan.load_state_dict(st2)
    st3 = plan.state_dict()
    assert sorted(st2) == sorted(st3) and all(np.array_equal(st2[k], st3[k]) for k in st2)
    assert not fails, "\n".join(fails[:20])
  finally:
    _lib.set_plane_format(before)


# ------------------------------------------------------------------------------------------------------------------
# Estimator: the example builder over three iterations against the float64 reference
# ------------------------------------------------------------------------------------------------------------------
EB, ED, EC, E_STEPS, WIDTH = 256, 20, 4, 6, 16


def _generator():
  import adanet_b200 as adanet
  from adanet_b200 import graph, train

  class Ex(adanet.subnetwork.Builder):
    def __init__(self, t, k):
      self.t, self.k = t, k

    @property
    def name(self):
      return "ex%d" % self.k

    def build_subnetwork(self, features, logits_dimension, training, iteration_step, summary, previous_ensemble=None):
      x = graph.input_layer(features, [graph.numeric_column("x", ED)])
      h = graph.dense(x, WIDTH + 8 * self.k, activation=graph.relu,
                      kernel_initializer=graph.glorot_uniform_initializer(100 * self.t + self.k))
      if previous_ensemble:
        h = graph.concat([h, previous_ensemble.weighted_subnetworks[-1].subnetwork.shared["hidden"]], axis=-1)
      logits = graph.dense(h, logits_dimension, kernel_initializer=graph.glorot_uniform_initializer(100 * self.t + self.k + 50))
      return adanet.Subnetwork(last_layer=h, logits=logits, complexity=1.0 + self.k, shared={"hidden": h})

    def build_subnetwork_train_op(self, subnetwork, loss, var_list, labels, iteration_step, summary, previous_ensemble):
      return train.MomentumOptimizer(0.05, 0.9).minimize(loss, var_list)

  class Gen(adanet.subnetwork.Generator):
    def generate_candidates(self, previous_ensemble, iteration_number, previous_ensemble_reports, all_reports):
      return [Ex(iteration_number, k) for k in range(2)]

  return Gen()


def _estimator(model_dir, mix, save_every=None, record=None):
  import adanet_b200 as adanet
  from adanet_b200 import train
  est = adanet.Estimator(
      head=adanet.heads.MultiClassHead(EC), subnetwork_generator=_generator(), max_iteration_steps=E_STEPS,
      ensemblers=[adanet.ensemble.ComplexityRegularizedEnsembler(optimizer=train.GradientDescentOptimizer(0.01),
                                                                 mixture_weight_type=mix, adanet_lambda=0.01)],
      max_iterations=3, model_dir=model_dir, config=adanet.RunConfig(model_dir=model_dir, save_checkpoints_steps=save_every),
      debug=True)
  if record is not None:
    inner = est._search_space

    def space(t, frozen):
      specs = inner(t, frozen)
      record[t] = [co.ConnectedSpec(s.name, s.dims, s.complexity, s.optimizer, ws=[w.copy() for w in s.ws],
                                    bs=[b.copy() for b in s.bs], inputs=s.inputs) for s in specs]
      return specs
    est._search_space = space
  return est


def _input(x, y, start=0):
  def fn():
    for i in range(start * EB, x.shape[0] - EB + 1, EB):
      yield {"x": x[i:i + EB]}, y[i:i + EB]
  return fn


def _match_oracle(s, res):
  """winners, architecture and every candidate's per-step sub_loss / adanet_loss / EMA against the reference, to the
  bound of the project's other Estimator parity tests (tests/test_gpu_api.py)"""
  assert len(s.reports) == len(res)
  for rep, r in zip(s.reports, res):
    assert rep.best_index == r.best_index and rep.candidate_names[1:] == r.candidate_names[1:]
    assert [tuple(a) for a in rep.architecture] == [tuple(a) for a in r.architecture]
    np.testing.assert_allclose(rep.ema_losses, r.ema_losses, atol=1e-5, rtol=0)
    for nm, tr in r.traces.items():
      for f in ("sub_loss", "adanet_loss", "ema"):
        np.testing.assert_allclose(rep.traces[nm][f], tr[f], atol=1e-5, rtol=0, err_msg="%s %s" % (nm, f))


def _check_inference(model_dir, mix, frozen, res, x, y):
  """predict / evaluate from a fresh Estimator on the model_dir against the reference's final ensemble"""
  want = co.ensemble_logits(frozen, mix, res[-1].mixture_weights, res[-1].bias, x[:EB])
  preds = list(_estimator(model_dir, mix).predict(lambda: iter([({"x": x[:EB]}, y[:EB])]), yield_single_examples=False))
  got = np.concatenate([np.asarray(p["logits"]) for p in preds], axis=0)[:EB]
  np.testing.assert_allclose(got, want, atol=2e-5, rtol=0)
  metrics = _estimator(model_dir, mix).evaluate(lambda: iter([({"x": x[:EB]}, y[:EB])]), steps=1)
  loss, _ = orc.softmax_xent_mean(want, y[:EB])
  assert abs(float(metrics["average_loss"]) - float(loss)) < 1e-5


def _same_dir(a, b):
  with np.load(os.path.join(a, "ensemble-latest.npz")) as p, np.load(os.path.join(b, "ensemble-latest.npz")) as q:
    assert sorted(p.files) == sorted(q.files)
    for k in q.files:
      assert np.array_equal(p[k], q[k]), k
  with open(os.path.join(a, "ensemble-latest.json")) as f, open(os.path.join(b, "ensemble-latest.json")) as g:
    assert json.load(f) == json.load(g)


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["scalar", "vector"])
def test_estimator_connected_search_matches_oracle(tmp_path, mix):
  from tests.test_gpu_plane_groups import _open
  _open()
  x, y = orc.make_tabular(EB * 3 * E_STEPS, ED, EC, seed=99)
  full_dir = str(tmp_path / "full")
  record = {}
  est = _estimator(full_dir, mix, record=record)
  est.train(_input(x, y), max_steps=3 * E_STEPS)
  s = est._search
  assert s.iteration == 3
  # the reference over the same initial weights and piece lists
  ens = orc.EnsemblerSpec(optimizer=("sgd", 0.01), mixture_weight_type=mix, adanet_lambda=0.01)
  assert record[0][0].optimizer[0] == "momentum"     # piece slots go through the in-flight resume below
  res, frozen = co.run_adanet(lambda t, fr: record[t], x, y, EB, E_STEPS, 3, ens, EC)
  _match_oracle(s, res)
  assert any(f.inputs for f in s.frozen[1:]), "no frozen member reads another one"
  with open(os.path.join(full_dir, "ensemble-latest.json")) as f:
    meta = json.load(f)
  assert [m.get("inputs") is not None for m in meta["members"]] == [f.inputs is not None for f in frozen]
  assert meta["members"][-1]["shared"]["hidden"]["__adanet_layer__"][0][:2] == [frozen[-1].iteration, frozen[-1].name]
  # evaluate / predict from a fresh Estimator on the model_dir
  _check_inference(full_dir, mix, frozen, res, x, y)
  # killed at an iteration boundary, resumed by a fresh Estimator
  kdir = str(tmp_path / "kill")
  _estimator(kdir, mix).train(_input(x, y), max_steps=E_STEPS)
  _estimator(kdir, mix).train(_input(x, y, E_STEPS), max_steps=3 * E_STEPS)
  _same_dir(kdir, full_dir)
  # killed inside iteration 1 after an in-flight save at global step 9, resumed from it
  idir = str(tmp_path / "inflight")
  a = _estimator(idir, mix, save_every=3)
  a.train(_input(x, y), max_steps=E_STEPS + 4)
  _estimator(idir, mix, save_every=3).train(_input(x, y, E_STEPS + 3), max_steps=3 * E_STEPS)
  _same_dir(idir, full_dir)


@pytest.mark.gpu
def test_tf32_fallback_in_an_iteration_with_pieces(tmp_path):
  """Iteration 2's first batch overflows fp16.  Its frozen members include a connected one, whose hidden and piece
  weight planes ensure_format re-creates on TF32; the re-run reads them through fresh fwd_op / backward pointers.  The
  run then matches the reference fed the batches the run kept (the discarded attempt's are left out)."""
  from adanet_b200 import _lib
  from tests.test_gpu_plane_groups import _open
  from tests.test_gpu_search_boundary import SPIKE
  _open()
  before = _lib.plane_format()
  _lib.set_plane_format(_lib.PLANES_F16)
  _lib.plane_overflow()
  try:
    x, y = orc.make_tabular(EB * 4 * E_STEPS, ED, EC, seed=77)
    x = x.copy()
    x[2 * E_STEPS * EB, 3] = SPIKE          # row 0 of iteration 2's first batch
    record = {}
    est = _estimator(str(tmp_path / "run"), "scalar", record=record)
    est.train(_input(x, y), max_steps=3 * E_STEPS)
    s = est._search
    assert s.tf32_fallbacks == 1 and _lib.plane_format() == _lib.PLANES_TF32 and s.iteration == 3
    assert any(f.inputs for f in s.frozen), "no connected member was frozen across the fallback"
    keep = np.r_[0:2 * E_STEPS * EB, 3 * E_STEPS * EB:4 * E_STEPS * EB]
    ens = orc.EnsemblerSpec(optimizer=("sgd", 0.01), mixture_weight_type="scalar", adanet_lambda=0.01)
    res, frozen = co.run_adanet(lambda t, fr: record[t], x[keep], y[keep], EB, E_STEPS, 3, ens, EC)
    _match_oracle(s, res)
    _check_inference(str(tmp_path / "run"), "scalar", frozen, res, x[keep], y[keep])
  finally:
    _lib.set_plane_format(before)
    _lib.plane_overflow()


@pytest.mark.gpu
def test_piece_optimizer_slots_round_trip():
  """Momentum slots of every piece: a plan restored from another plan's state_dict takes the same next step, byte for
  byte."""
  import torch
  from adanet_b200.core import engine as eng
  from tests.test_gpu_plane_groups import _open
  _open()
  rng = np.random.default_rng(3)
  plan, fnets, _ = _build(rng)
  specs = [eng.SubnetworkPlanSpec(c.spec.name, c.spec.dims, 2.0, ("momentum", LR, 0.9), [w.copy() for w in c.spec.ws],
                                  [b.copy() for b in c.spec.bs], dropout=c.spec.dropout, inputs=c.spec.inputs)
           for c in plan.candidates]
  dev = torch.device("cuda", torch.cuda.current_device())
  mk = lambda: eng.IterationPlan(2, specs, fnets, eng.EnsemblerPlanSpec(**ENS), B, D, C, "softmax_xent", device=dev)
  a = mk()
  x, y = orc.make_tabular(B * 4, D, C, seed=8)
  for k in range(3):
    a.train_step(x[k * B:(k + 1) * B], y[k * B:(k + 1) * B])
  sa = a.state_dict()
  assert any(k.startswith("c2_sub_opt_s0_") for k in sa)
  n_slots = len([k for k in sa if k.startswith("c2_sub_opt_s0_")])
  assert n_slots == 2 + 3 + 1, n_slots        # layer 0 (w, b), layer 1 as three pieces + its bias
  b = mk()
  b.load_state_dict(sa)
  sb = b.state_dict()
  assert all(np.array_equal(sa[k], sb[k]) for k in sa)
  a.train_step(x[3 * B:], y[3 * B:])
  b.train_step(x[3 * B:], y[3 * B:])
  sa, sb = a.state_dict(), b.state_dict()
  assert sorted(sa) == sorted(sb)
  for k in sa:
    if k != "steps_done":
      assert np.array_equal(sa[k], sb[k]), k


# ------------------------------------------------------------------------------------------------------------------
# Two ranks on one GPU over gloo: the winner of iterations 0 and 1 is owned by rank 1, so rank 0 builds its replica of
# a connected member from the spec, against its own frozen list, and re-splits the piece planes after the broadcast
# ------------------------------------------------------------------------------------------------------------------
R_B, R_STEPS = 256, 4


def _rank_space(t, frozen):
  from adanet_b200.core import engine as eng
  out = []
  for k, w in enumerate((256, 24)):        # the wide candidate goes to rank 0, the narrow one to rank 1
    rng = np.random.default_rng(1000 * t + k)
    inputs = None
    dims = [D, w, C]
    if frozen:
      f = frozen[-1]
      hw = f.dims[1]
      inputs = [None, [_own(0, w), _mem(f.iteration, f.name, 0, w, w + hw)]]
    ws, bs = _params(rng, dims, inputs)
    out.append(eng.SubnetworkPlanSpec("r%d" % k, dims, 1.0 + k, ("momentum", 0.05, 0.9), ws, bs, inputs=inputs))
  return out


def _two_rank_worker(rank, world, port, q):
  import datetime
  import torch
  import torch.distributed as dist
  os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
  torch.cuda.set_device(0)
  dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=60))
  out = dict(fails=[], replicas=[], losses=[], logits=None)
  try:
    from adanet_b200.core import engine as eng
    from adanet_b200.core import search as srch
    from tests.test_gpu_plane_groups import _open
    _open()
    x, y = orc.make_tabular(R_B * R_STEPS * 3, D, C, seed=21)
    s = srch.AdaNetSearch(_rank_space, eng.EnsemblerPlanSpec(**ENS), D, C, R_B, placement="balanced",
                          replay_indices=[1, 2, 2])
    batches = srch.consecutive_batches(x, y, R_B)
    for t in range(3):
      s.build_iteration()
      if t < 2 and s._owners != [0, 1]:
        out["fails"].append("iteration %d: owners %s, want [0, 1]" % (t, s._owners))
      secs = s.train_iteration(batches, R_STEPS)
      rep = s.finish_iteration(secs)
      out["losses"].append([float(v) for v in rep.ema_losses])
      reps = []
      for f in s.frozen:
        ws, bs = f.numpy_params()
        reps += ws + bs
        # the hi / lo words of every piece's planes (a weight's sign-bit words are never read)
        reps += [wp[:st._planes_words(r1 - r0, f.dims[i + 1])].cpu().numpy() for i in range(len(f.ws))
                 for (r0, r1), wp in zip(f.piece_rows(i), f.piece_wps[i])]
      out["replicas"].append(reps)
    if not any(f.inputs for f in s.frozen):
      out["fails"].append("no connected member was frozen")
    ev = eng.EnsembleEvalPlan(s.frozen, s.mixture_weights, s.bias, s.winner_ens, "softmax_xent", R_B, C)
    ev.run(x[:R_B], y[:R_B])
    out["logits"] = ev.ens_logits.cpu().numpy()
  except Exception as e:        # reported, not raised: the parent process checks it
    import traceback
    out["fails"].append("rank %d: %s" % (rank, traceback.format_exc()))
  finally:
    q.put((rank, out))
    dist.destroy_process_group()


@pytest.mark.gpu
def test_two_ranks_replicate_connected_winners():
  import torch.multiprocessing as mp
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = st._free_port()
  procs = [ctx.Process(target=_two_rank_worker, args=(r, 2, port, q)) for r in range(2)]
  for p in procs:
    p.start()
  got = {}
  try:
    for _ in procs:
      rank, out = q.get(timeout=300)
      got[rank] = out
  finally:
    for p in procs:
      p.join(timeout=60)
      if p.is_alive():
        p.kill()
        p.join()
  fails = [f for r in sorted(got) for f in got[r]["fails"]]
  assert not fails, "\n".join(fails)
  a, b = got[0], got[1]
  assert a["losses"] == b["losses"]
  for t, (ra, rb) in enumerate(zip(a["replicas"], b["replicas"])):
    assert len(ra) == len(rb) and all(np.array_equal(u, v) for u, v in zip(ra, rb)), "iteration %d replicas differ" % t
  assert np.array_equal(a["logits"], b["logits"])
