"""The state AdaNetSearch hands from one iteration to the next (core/search.py finish_iteration -> build_iteration,
core/engine.py EnsembleHead.__init__ and DenseNet.ensure_format / refresh_planes), element by element.

The per-step losses of test_gpu_iteration / test_gpu_multi / test_gpu_api cannot see state that barely moves the loss: a
warm-start row of a member with a small weight, weight planes split from stale weights or in the old format, a bias
that was not carried over.  Every case here drives the search itself for three iterations and, at every boundary
t -> t + 1:

  (a) copies to the host every local candidate's final weights, each head's mixture weights, bias and EMA state, and
      the frozen members, before finish_iteration;
  (b) checks the plan of t + 1 before its first step, exactly: the frozen members are the kept previous ones in kept
      order, then the winner's new ones, byte-equal to (a); every frozen plane buffer is a fresh split of its weights in
      the CURRENT format (K padding included, a conv stem's stem_out sized for it); architecture, replay trace, winning
      ensembler and prev_best_ema follow the selection rules; every head starts from the mixture weights and bias that
      weighted.py gives (1/N, zeros for MATRIX, initial_weight_fn, the winner's warm-start rows of the kept members for
      the winner's ensembler only, MeanEnsembler zeros and 1/n_new), restated in float64; the candidates start from
      their specs' weights; optimizer slots, step counters, step_dev, EMA and trace are zero;
  (c) teacher-forces the first two steps of t + 1 with the checkers of test_gpu_step_state, the frozen members' float64
      forward taken from (a) -- not from the plan -- so a member frozen from the wrong or pre-final-step weights, from
      stale or old-format planes, or replayed with dropout fails there.

The TF32 fallback at t = 1 (a feature value of 7e4 in one row of iteration 1's first batch) must rebuild a plan that
passes (b) against the same boundary copy, every frozen member -- a conv-stem one included -- re-split into TF32 planes,
and (c) on the batches after the discarded attempt.  At the Estimator level, a run that falls back while saving
in-flight checkpoints, and runs killed after the fallback and resumed in a fresh fp16 process, end byte-identical to
the uninterrupted run.  The worst err/bound of every stage of (c) is printed at the end of the module (pytest -s).
"""

import json
import os

import numpy as np
import pytest

from tests.parity_util import orc
from tests import test_gpu_step_state as st

D = 100
ENS = dict(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001)
STEPS = 3              # per iteration: two teacher-forced steps, then one plain one
ITERS = 3
SPIKE = 7e4            # beyond fp16's 65504: the input split raises the overflow flag


def _lin(C, opt=("sgd", 0.05)):
  return dict(dims=[D, C], opt=opt)


def _hid(C, w=40, opt=("momentum", 0.02, 0.9), **kw):
  return dict(dims=[D, w, C], opt=opt, **kw)


def _keep_0_2(specs, n_frozen):
  """partial pruning once three members are frozen: the first candidate keeps members [0, 2]; before that, the All
  strategy grows the three new subnetworks at once"""
  from adanet_b200.core import search as srch
  if n_frozen >= 3:
    return [srch.EnsembleCandidate("n0_prune", [0], [0, 2]), srch.EnsembleCandidate("n1_grow", [1], True)]
  return [srch.EnsembleCandidate("all", [0, 1, 2], True), srch.EnsembleCandidate("n0_grow", [0], True)]


VEC_WARM = dict(optimizer=("adam", 0.01), mixture_weight_type="vector", use_bias=True, adanet_lambda=0.02,
                adanet_beta=0.003, warm_start_mixture_weights=True)
CASES = {
    "grow_scalar": dict(B=256, C=10, head="softmax_xent", ens=[ENS], cands=[_hid(10), _lin(10)]),
    "vector_warm": dict(B=256, C=10, head="softmax_xent", ens=[VEC_WARM],
                        cands=[_hid(10, 64, ("sgd", 0.05)), dict(dims=[D, 40, 130, 10], opt=("adam", 0.01))]),
    "vector_warm_legacy": dict(B=256, C=10, head="softmax_xent", ens=[dict(VEC_WARM, legacy_train_op=True)],
                               cands=[_hid(10, 64, ("sgd", 0.05)), _lin(10, ("rmsprop", 0.01))]),
    # a linear winner at t = 0 (its last layer is the minibatch's own planes), a hidden one at t = 1
    "matrix_warm": dict(B=256, C=10, head="softmax_xent", replay=[0, 2, 1],
                        ens=[dict(optimizer=("sgd", 0.05), mixture_weight_type="matrix", use_bias=True, adanet_lambda=0.01,
                                  adanet_beta=0.001, warm_start_mixture_weights=True)],
                        cands=[_lin(10), _hid(10, 48)]),
    # the previous ensemble kept at t = 1, grown at t = 2
    "replay_keep": dict(B=256, C=10, head="softmax_xent", replay=[1, 0, 2], ens=[dict(VEC_WARM, mixture_weight_type="scalar")],
                        cands=[_hid(10), _lin(10)]),
    "force_grow": dict(B=37, C=10, head="softmax_xent", force_grow=True, ens=[dict(ENS, use_bias=True)], cands=[_hid(10, 72)]),
    # All (three new members at once) at t = 0, then a candidate that keeps members [0, 2] of 3 wins, warm-started
    "prune": dict(B=256, C=10, head="softmax_xent", replay=[0, 1, 2], candidates_fn=_keep_0_2, ens=[VEC_WARM],
                  cands=[_hid(10, 32), _lin(10), _hid(10, 24, ("sgd", 0.05))]),
    # a Solo winner at t = 1: nothing is kept
    "solo": dict(B=256, C=10, head="softmax_xent", replay=[0, 3, 2], strategies=("grow", "solo"), ens=[VEC_WARM],
                 cands=[_hid(10), _lin(10)]),
    # two ensemblers over every candidate: the second one's candidates win
    "two_ensemblers": dict(B=256, C=10, head="softmax_xent", replay=[1, 4, 2],
                           ens=[dict(ENS, warm_start_mixture_weights=True),
                                dict(VEC_WARM, optimizer=("momentum", 0.01, 0.9), name="second")],
                           cands=[_hid(10), _lin(10)]),
    # a MeanEnsembler winner, then a complexity-regularized one
    "mean_then_cr": dict(B=256, C=10, head="softmax_xent", replay=[1, 1, 2],
                         ens=[dict(VEC_WARM), dict(kind="mean", name="mean")], cands=[_hid(10), _lin(10)]),
    "dropout": dict(B=256, C=10, head="softmax_xent", replay=[0, 1, 1], ens=[dict(ENS, use_bias=True)],
                    cands=[dict(dims=[D, 64, 48, 10], opt=("sgd", 0.05), dropout=[(0.25, 7), (0.5, 9)]), _lin(10)]),
    "bagged": dict(B=256, C=10, head="softmax_xent", replay=[0, 1, 1], ens=[dict(ENS, use_bias=True)],
                   cands=[dict(dims=[D, 48, 40, 10], opt=("sgd", 0.05), dropout=[(0.25, 5), None], own=True),
                          _hid(10, 64)]),
    # SimpleCNN members on 8x8x3 images: a frozen conv stem replays into its own stem_out planes
    "cnn": dict(B=128, C=10, head="softmax_xent", input=192, replay=[0, 1, 2], ens=[ENS],
                cands=[dict(dims=[256, 32, 10], image=(8, 8, 3), opt=("momentum_cosine", 0.05, 0.9, 20, 0.1)),
                       dict(dims=[192, 40, 10], opt=("sgd", 0.05))]),
    # a custom mixture_weight_initializer (weighted.py:360-366)
    "mse": dict(B=256, C=3, head="mse", ens=[dict(ENS, use_bias=True, initial_weight_fn=lambda n, d, c: 0.7 / n)],
                cands=[_hid(3, 72), _lin(3, ("adam", 0.01))]),
    "sigmoid": dict(B=256, C=1, head="sigmoid_xent", ens=[dict(VEC_WARM)], cands=[_hid(1, 40, ("rmsprop", 0.01)), _lin(1)]),
}
SIMT_CASES = ["force_grow", "grow_scalar", "mse", "replay_keep", "sigmoid", "vector_warm", "vector_warm_legacy"]


# ------------------------------------------------------------------------------------------------------------------
# the search of a case
# ------------------------------------------------------------------------------------------------------------------
def _cand_descs(case, t):
  """the candidates of iteration t with their initial weights (glorot kernels, random biases; seed 1000 + 100 t + i)"""
  out = []
  for i, c in enumerate(case["cands"] if t == 0 else case.get("cands_later", case["cands"])):
    rng = np.random.default_rng(1000 + 100 * t + i)
    dims = c["dims"]
    ws = [orc.glorot_uniform(rng, dims[j], dims[j + 1]) for j in range(len(dims) - 1)]
    bs = [(rng.standard_normal(dims[j + 1]) * 0.1).astype(np.float32) for j in range(len(dims) - 1)]
    if c.get("image"):
      cin, f = c["image"][2], dims[0] // ((c["image"][0] // 2) * (c["image"][1] // 2))
      ws = [(rng.standard_normal((3, 3, cin, f)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)] + ws
      bs = [(rng.standard_normal(f) * 0.1).astype(np.float32)] + bs
    out.append(dict(c, name="n%d" % i, cx=float(np.sqrt(np.float32(len(dims) - 2))), p=(ws, bs)))
  return out


def _space(case):
  from adanet_b200.core import engine as eng

  def fn(t, frozen):
    return [eng.SubnetworkPlanSpec(c["name"], c["dims"], c["cx"], c["opt"], [w.copy() for w in c["p"][0]],
                                   [b.copy() for b in c["p"][1]], dropout=c.get("dropout"), image_shape=c.get("image"),
                                   own_input=c.get("own", False)) for c in _cand_descs(case, t)]
  return fn


def _search(case):
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  return srch.AdaNetSearch(_space(case), [eng.EnsemblerPlanSpec(**e) for e in case["ens"]], case.get("input", D), case["C"],
                           case["B"], head=case["head"], force_grow=case.get("force_grow", False),
                           replay_indices=case.get("replay"), strategies=case.get("strategies", ("grow",)),
                           candidates_fn=case.get("candidates_fn"), placement=case.get("placement", "balanced"))


def _step_case(case, s):
  """the case description teacher_forced_step reads: the heads of the plan as (name, builders, keep, -) by global index"""
  return dict(case, heads=[(c.name, list(c.builders), c.keep_previous, None) for c in s._ecands])


def _plain_step(case, plan, k):
  x, y = st._batch(case, k)
  own = {c.index: st._batch(case, 500 + k) for c in plan.candidates if c.bagged}
  plan.train_step(x, y, own_batches=own or None)


# ------------------------------------------------------------------------------------------------------------------
# (a) the boundary copy and what the rules make of it
# ------------------------------------------------------------------------------------------------------------------
def snapshot(s):
  """(a): the final state of every local candidate and head, and the frozen members, as host copies"""
  import torch
  torch.cuda.synchronize()
  plan = s.plan
  return dict(
      cands={c.index: tuple([a.copy() for a in p] for p in c.net.numpy_params()) for c in plan.candidates},
      heads={g: dict(mix=[t.cpu().numpy().copy() for t in h.mixture_weight_tensors()], bias=h.bias.cpu().numpy().copy(),
                     ema=h.ema_state.cpu().numpy().copy()) for g, h, _ in plan.heads},
      ema_losses=list(plan.ema_losses()),
      frozen=[dict(name=f.name, dims=list(f.dims), cx=f.complexity, it=f.iteration, image=f.image_shape,
                   p=tuple([a.copy() for a in p] for p in f.numpy_params())) for f in s.frozen])


def _best_index(losses, t, force_grow, replay):
  """the selection rule (adanet/core/estimator.py:1415-1517), restated: a replayed index; else np.nanargmin over the
  EMA losses, the previous ensemble (index 0 after the first iteration) left out under force_grow"""
  if replay is not None:
    return int(replay)
  a = np.asarray(losses, dtype=np.float32)
  if t > 0 and force_grow and len(a) > 1:
    return 1 + int(np.nanargmin(a[1:]))
  return int(np.nanargmin(a))


def _kept(keep_previous, n_frozen):
  """previous members a candidate keeps: True -> all, False / None -> none, else the listed ones"""
  if keep_previous is True:
    return list(range(n_frozen))
  return [] if keep_previous in (False, None) else [int(i) for i in keep_previous]


def expected_next(s, snap, prev, t):
  """the search state after finish_iteration(t) by the rules of adanet/core/estimator.py:1415-1517 and
  iteration.py:568-579, from the boundary copy (of every rank's heads, merged, on a multi-rank search)"""
  ecs = s._ecands
  losses = [float(snap["heads"][g]["ema"][2]) for g in range(len(ecs))]
  assert losses == [float(v) for v in snap["ema_losses"]]
  if t > 0:
    losses = [prev["prev_best_ema"]] + losses
  replay = s.replay_indices[t] if (s.replay_indices is not None and t < len(s.replay_indices)) else None
  best = _best_index(losses, t, s.force_grow, replay)
  out = dict(prev, replay_trace=prev["replay_trace"] + [best], best=best)
  if t > 0 and best == 0:
    return out
  ci = best - (1 if t > 0 else 0)
  ec = ecs[ci]
  kidx = _kept(ec.keep_previous, len(prev["frozen"]))
  new = [dict(name=s._specs[b].name, dims=list(s._specs[b].dims), cx=s._specs[b].complexity, it=t,
              image=s._specs[b].image_shape, p=snap["cands"][b]) for b in ec.builders]
  out.update(frozen=[prev["frozen"][i] for i in kidx] + new,
             architecture=[prev["architecture"][i] for i in kidx] + [(t, s._specs[b].name) for b in ec.builders],
             mix=snap["heads"][ci]["mix"], bias=snap["heads"][ci]["bias"], prev_best_ema=float(snap["heads"][ci]["ema"][2]),
             winner_ens=ec.ens_index)
  return out


def initial_head(mix_type, kind, n_prev, last_dims, C, warm_mix=None, warm_bias=None, init_fn=None):
  """float64 mixture weights and bias a candidate ensemble starts from (weighted.py:270-285,360-366,419-428,487-516;
  mean.py:92-135): SCALAR [N] / VECTOR [N, C] at 1/N or MATRIX [D_k, C] zeros; a custom initializer's value per member;
  the MeanEnsembler's 0 for kept and 1/n_new for new members; else the warm-start rows of the kept members and the bias"""
  N = len(last_dims)
  if mix_type == "matrix":
    mix = [np.zeros((d, C)) for d in last_dims]
  else:
    mix = np.full((N,) if mix_type == "scalar" else (N, C), float(np.float32(1.0 / N)))
  if init_fn is not None and kind != "mean":
    for k, d in enumerate(last_dims):
      w0 = np.asarray(init_fn(N, d, C), dtype=np.float32).astype(np.float64)
      mix[k] = w0.reshape(np.shape(mix[k]))
  bias = np.zeros(C)
  if kind == "mean":
    mix[:] = 0.0
    mix[n_prev:] = float(np.float32(1.0 / (N - n_prev)))
  elif warm_mix is not None and n_prev > 0:
    for k in range(n_prev):
      mix[k] = np.asarray(warm_mix[k], dtype=np.float64).reshape(np.shape(mix[k]))
    if warm_bias is not None:
      bias = np.asarray(warm_bias, dtype=np.float64).reshape(C)
  return mix, bias


def _bytes(a):
  a = np.ascontiguousarray(a)
  return a.view(np.uint8) if a.size else a


def _same(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(_bytes(a), _bytes(b))


def check_boundary(fails, s, exp, t, case):
  """(b) on the plan of iteration t just built"""
  import torch
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  plan = s.plan
  tag = "boundary %d -> %d" % (t - 1, t)
  # the search's own record
  if s.architecture != exp["architecture"]:
    fails.append("%s: architecture %s, want %s" % (tag, s.architecture, exp["architecture"]))
  if s.replay_trace != exp["replay_trace"]:
    fails.append("%s: replay trace %s, want %s" % (tag, s.replay_trace, exp["replay_trace"]))
  if s.winner_ens_index != exp["winner_ens"]:
    fails.append("%s: winning ensembler %d, want %d" % (tag, s.winner_ens_index, exp["winner_ens"]))
  if s.prev_best_ema != exp["prev_best_ema"]:
    fails.append("%s: prev_best_ema %r, want %r" % (tag, s.prev_best_ema, exp["prev_best_ema"]))
  got_mix = s.mixture_weights if isinstance(s.mixture_weights, list) else [s.mixture_weights]
  if len(got_mix) != len(exp["mix"]) or not all(_same(a, b) for a, b in zip(got_mix, exp["mix"])) or not _same(s.bias, exp["bias"]):
    fails.append("%s: the search's mixture weights / bias are not the winner's final ones" % tag)
  # frozen members: kept ones in kept order, then the winner's new ones, byte-equal to the boundary copy
  names = [f.name for f in s.frozen]
  if names != [f["name"] for f in exp["frozen"]] or plan.frozen != s.frozen:
    fails.append("%s: frozen members %s, want %s" % (tag, names, [f["name"] for f in exp["frozen"]]))
    return
  fmt = _lib.plane_format()
  for j, (f, e) in enumerate(zip(s.frozen, exp["frozen"])):
    ws, bs = f.numpy_params()
    if f.iteration != e["it"] or list(f.dims) != e["dims"] or f.complexity != e["cx"]:
      fails.append("%s: frozen %d (%s): iteration / dims / complexity" % (tag, j, f.name))
    if not all(_same(a, b) for a, b in zip(ws + bs, e["p"][0] + e["p"][1])) or len(ws) != len(e["p"][0]):
      fails.append("%s: frozen %d (%s): weights differ from the winner's final ones" % (tag, j, f.name))
    if f.planes:
      if f.fmt != fmt:
        fails.append("%s: frozen %d (%s) still in plane format %d" % (tag, j, f.name, f.fmt))
      for i, wp in enumerate(f.wps):
        if wp.numel() != eng.new_planes(f.dims[i], f.dims[i + 1], f.device).numel():
          fails.append("%s: frozen %d (%s) W%d planes are sized for another format" % (tag, j, f.name, i))
      for i, hp in enumerate(f.hp):
        if hp.numel() != eng.new_planes(f.batch, f.dims[i + 1], f.device).numel():
          fails.append("%s: frozen %d (%s) hidden planes %d are sized for another format" % (tag, j, f.name, i))
      if f.stem and f.stem_out.numel() != eng.new_planes(f.batch, f.dims[0], f.device).numel():
        fails.append("%s: frozen %d (%s) stem_out is sized for another format" % (tag, j, f.name))
      sub = []
      st.check_planes_resplit(sub, [("W%d" % i, w, wp) for i, (w, wp) in enumerate(zip(f.ws, f.wps))], "")
      if sub:
        fails.append("%s: frozen %d (%s): its weight planes are not a split of its weights%s" % (tag, j, f.name, sub[0]))
  # every head: the mixture weights and bias it starts from
  winner_name = s.ensemblers[exp["winner_ens"]].name
  nf = len(s.frozen)
  for g, h, _ in plan.heads:
    ec = s._ecands[g]
    e = s.ensemblers[ec.ens_index]
    kidx = _kept(ec.keep_previous, nf)
    members = [s.frozen[i] for i in kidx] + [s._specs[b] for b in ec.builders]
    warm = bool(e.warm_start_mixture_weights) and e.kind != "mean" and e.name == winner_name and exp["mix"] is not None
    prev_mix = exp["mix"] if e.mixture_weight_type == "matrix" else exp["mix"][0]
    want_mix, want_bias = initial_head(e.mixture_weight_type, e.kind, len(kidx), [m.dims[-2] for m in members], s.C,
                                       [prev_mix[i] for i in kidx] if warm else None, exp["bias"] if warm else None,
                                       e.initial_weight_fn)
    got = [t_.cpu().numpy() for t_ in h.mixture_weight_tensors()]
    want = want_mix if e.mixture_weight_type == "matrix" else [want_mix]
    for k, (a, b) in enumerate(zip(got, want)):
      if a.shape != b.shape or not np.array_equal(a.astype(np.float64), b):
        fails.append("%s head %s: initial mixture weights %d\n%s\nwant\n%s" % (tag, h.name, k, a, b))
    if not np.array_equal(h.bias.cpu().numpy().astype(np.float64), want_bias):
      fails.append("%s head %s: initial bias %s, want %s" % (tag, h.name, h.bias.cpu().numpy(), want_bias))
    if e.mixture_weight_type == "matrix":
      st.check_planes_resplit(fails, [("mixture weight %d" % k, w, wp) for k, (w, wp) in enumerate(zip(h.mw, h.mwp))],
                              "%s head %s" % (tag, h.name))
  # everything that trains starts from its spec and from zero
  stt = plan.state_dict()
  if int(stt["step_dev"]) != 0 or int(stt["steps_done"]) != 0:
    fails.append("%s: step_dev / steps_done not zero" % tag)
  kinds = {}
  for c in plan.candidates:
    sp = s._specs[c.index]
    kinds["c%d_sub_opt_" % c.index] = sp.optimizer[0]
    ws, bs = c.net.numpy_params()
    if not all(_same(a, np.asarray(b, np.float32)) for a, b in zip(ws + bs, list(sp.ws) + list(sp.bs))):
      fails.append("%s: candidate %d does not start from its spec's weights" % (tag, c.index))
  for g, h, _ in plan.heads:
    if h.ens_opt is not None:
      kinds[st._head_key(plan, g, h) + "ens_opt_"] = h.ens.optimizer[0]
  for key, v in stt.items():
    pre = next((p for p in kinds if key.startswith(p)), None)
    if pre is not None:
      slot = key[len(pre):]
      if slot == "step":
        ok = int(v) == 0
      else:
        want = st._fresh_slots(kinds[pre], v)[0 if slot.startswith("s0") else 1]
        ok = want is not None and np.array_equal(v, want)
      if not ok:
        fails.append("%s: %s does not start fresh" % (tag, key))
    elif key.endswith("ema_state") or key.endswith("trace"):
      if np.any(v != 0):
        fails.append("%s: %s not zero" % (tag, key))
  torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# driving a case
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", autouse=True)
def _report():
  saved = dict(st.REPORT)
  st.REPORT.clear()
  yield
  for f in sorted({f for f, _ in st.REPORT}):
    print("\nsearch boundary, %s planes: " % f + ", ".join("%s %.3g" % (sg, v) for (ff, sg), v in sorted(st.REPORT.items())
                                                          if ff == f and not sg.startswith("deep")))
  st.REPORT.clear()
  st.REPORT.update(saved)


def _forced_steps(case, s, exp, k0, fails):
  """(c): the first two steps of the plan just built, every stage against float64 with the frozen members of (a)"""
  plan = s.plan
  cands = _cand_descs(case, s.iteration)
  frozen = [dict(p=f["p"]) for f in exp["frozen"]]
  for j in range(2):
    st.teacher_forced_step(plan, plan.frozen, _step_case(case, s), frozen, [cands[c.index] for c in plan.candidates],
                           k0 + j, fails)
  return STEPS - 2


def run_case(case, name, spike_at=None):
  """ITERS iterations; (a) at every boundary, (b) and (c) on every plan after the first.  spike_at = t: row 0 of
  iteration t's first batch carries SPIKE, the iteration is discarded and re-run on TF32 planes from the same boundary"""
  import torch
  s = _search(case)
  exp = dict(frozen=[], architecture=[], replay_trace=[], mix=None, bias=None, prev_best_ema=None, winner_ens=0)
  fails = []
  fallbacks = 0
  for t in range(ITERS):
    s.build_iteration()
    k0 = 100 * t
    if t == spike_at:
      for j in range(STEPS):
        x, y = st._batch(case, k0 + j)
        if j == 0:
          x = x.copy()
          x[0, 3] = SPIKE
        own = {c.index: st._batch(case, 500 + k0 + j) for c in s.plan.candidates if c.bagged}
        s.plan.train_step(x, y, own_batches=own or None)
      assert s.restart_on_tf32_if_overflowed(), "%s: the spike did not raise the fp16 overflow flag" % name
      fallbacks += 1
      s.build_iteration()
      k0 += 50             # the re-run trains on the batches after the discarded attempt
    rest = STEPS
    if t > 0:
      check_boundary(fails, s, exp, t, case)
      assert not fails, "%s:\n%s" % (name, "\n".join(fails[:30]))
      rest = _forced_steps(case, s, exp, k0, fails)
      assert not fails, "%s:\n%s" % (name, "\n".join(fails[:30]))
    for j in range(STEPS - rest, STEPS):
      _plain_step(case, s.plan, k0 + j)
    assert not s.restart_on_tf32_if_overflowed(), "%s: iteration %d overflowed the fp16 planes" % (name, t)
    snap = snapshot(s)
    exp = expected_next(s, snap, exp, t)
    rep = s.finish_iteration()
    assert rep.best_index == exp["best"], "%s: iteration %d selected %d, want %d" % (name, t, rep.best_index, exp["best"])
  torch.cuda.synchronize()
  return s, fallbacks


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_search_boundaries(fmt, name):
  """Three iterations of each case; at both boundaries the next plan's state is exact (b) and its first two steps
  match float64 over the frozen members of the boundary copy (c)."""
  from adanet_b200 import _lib
  run_case(CASES[name], name)
  assert not _lib.plane_overflow()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SIMT_CASES)
def test_search_boundaries_simt(simt_path, name):
  """The same boundaries on the fp32 SIMT cross-check path (no planes: frozen members keep dense activations)."""
  run_case(CASES[name], name)


@pytest.fixture
def simt_path():
  from tests.test_gpu_plane_groups import _open
  _, _lib, _ = _open()
  _lib.set_dense_path(_lib.PATH_SIMT)
  yield
  _lib.set_dense_path(_lib.PATH_AUTO)


@pytest.fixture(scope="module", params=["f16", "tf32"])
def fmt(request):
  from tests.test_gpu_plane_groups import _open, _set_format
  _, _lib, _ = _open()
  before = _lib.plane_format()
  _set_format(_lib, request.param)
  _lib.plane_overflow()
  yield request.param
  _lib.set_plane_format(before)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cnn", "vector_warm", "matrix_warm"])
def test_tf32_fallback_after_the_first_iteration(name):
  """fp16 planes; the spike in iteration 1's first batch makes the search discard that iteration and switch to TF32:
  the rebuilt plan passes (b) against the boundary copy taken before the fp16 attempt -- every frozen member, the conv
  stem's stem_out included, re-split into TF32 planes -- and its first two steps (c); iteration 2 follows on TF32."""
  from tests.test_gpu_plane_groups import _open
  _, _lib, _ = _open()
  _lib.set_plane_format(_lib.PLANES_F16)
  _lib.plane_overflow()
  s, fallbacks = run_case(CASES[name], name, spike_at=1)
  assert fallbacks == 1 and _lib.plane_format() == _lib.PLANES_TF32
  assert all(f.fmt == _lib.PLANES_TF32 for f in s.frozen)


# ------------------------------------------------------------------------------------------------------------------
# two ranks: the handover between GPUs
# ------------------------------------------------------------------------------------------------------------------
MULTI = {
    # round robin over three candidates: rank 0 owns 0 and 2, rank 1 owns 1, which wins at t = 0 -- the gathered losses
    # must follow the owners, rank 0 gets the winner by broadcast and re-splits its planes
    "owner_rank1": dict(B=256, C=10, head="softmax_xent", placement="round_robin", replay=[1, 1], ens=[VEC_WARM],
                        cands=[_hid(10), _lin(10), _hid(10, 24, ("sgd", 0.05))]),
    # the heavy candidate is row-sharded over both ranks at t = 0 and wins: it is rebuilt at the full batch; t = 1 has two
    # light, whole candidates
    "sharded": dict(B=256, C=10, head="softmax_xent", placement="sharded", replay=[0, 1], ens=[dict(VEC_WARM)],
                    cands=[dict(dims=[D, 512, 512, 10], opt=("momentum", 0.02, 0.9)), _lin(10)],
                    cands_later=[_hid(10), _hid(10, 40, ("sgd", 0.05))]),
}


def _merged_snapshot(s):
  """(a) on every rank, merged: each candidate and head from a rank that holds it"""
  import torch.distributed as dist
  mine = snapshot(s)
  every = [None] * dist.get_world_size()
  dist.all_gather_object(every, mine)
  out = dict(cands={}, heads={}, frozen=mine["frozen"])
  for o in every:
    for k, v in o["cands"].items():
      out["cands"].setdefault(k, v)
    for k, v in o["heads"].items():
      out["heads"].setdefault(k, v)
  out["ema_losses"] = [float(out["heads"][g]["ema"][2]) for g in sorted(out["heads"])]
  return out


def _replicas(s):
  """what must be byte-identical on every rank after a boundary: the frozen members' weights and the hi / lo words of
  their weight planes (the sign-bit words of a weight are never read), the mixture weights and the bias"""
  out = []
  for f in s.frozen:
    ws, bs = f.numpy_params()
    out += ws + bs
    if f.planes:
      out += [wp[:st._planes_words(w.shape[0], w.shape[1])].cpu().numpy() for w, wp in zip(f.ws, f.wps)]
  mw = s.mixture_weights if isinstance(s.mixture_weights, list) else [s.mixture_weights]
  return out + [np.asarray(m) for m in mw] + [np.asarray(s.bias)]


def _rank_worker(rank, world, port, name, fmt_name, q):
  import datetime
  import torch
  import torch.distributed as dist
  os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
  timeout = datetime.timedelta(seconds=60)
  if torch.cuda.device_count() >= world:
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank), timeout=timeout)
  else:        # fewer GPUs than ranks: share cuda:0, exchange over gloo
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timeout)
  fails, replicas = [], []
  try:
    from tests.test_gpu_plane_groups import _open, _set_format
    _, _lib, _ = _open()
    _set_format(_lib, fmt_name)
    _lib.plane_overflow()
    case = MULTI[name]
    s = _search(case)
    exp = dict(frozen=[], architecture=[], replay_trace=[], mix=None, bias=None, prev_best_ema=None, winner_ens=0)
    for t in range(2):
      s.build_iteration()
      k0, rest = 100 * t, STEPS
      if t > 0:      # the steps run on whatever (b) found: the ranks stay in step through the next collectives
        check_boundary(fails, s, exp, t, case)
        rest = _forced_steps(case, s, exp, k0, fails)
      for j in range(STEPS - rest, STEPS):
        _plain_step(case, s.plan, k0 + j)
      snap = _merged_snapshot(s)
      exp = expected_next(s, snap, exp, t)
      rep = s.finish_iteration()
      got = [float(v) for v in rep.ema_losses[1 if t > 0 else 0:]]
      if got != snap["ema_losses"]:
        fails.append("iteration %d: gathered EMA losses %s, the owners' heads hold %s" % (t, got, snap["ema_losses"]))
      if rep.best_index != exp["best"]:
        fails.append("iteration %d: selected %d, want %d" % (t, rep.best_index, exp["best"]))
      replicas.append(_replicas(s))
      if t == 0 and name == "sharded" and not s._shard_ranks[0] == [0, 1]:
        fails.append("the heavy candidate was not row-sharded: %s" % (s._shard_ranks,))
  except Exception as e:        # reported, not raised: the parent process checks it
    fails.append("rank %d: %s: %s" % (rank, type(e).__name__, e))
  finally:
    q.put((rank, fails, replicas))
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MULTI))
def test_two_rank_boundary(fmt, name):
  """Two ranks (two processes sharing cuda:0 over gloo, or NCCL on two GPUs): on EVERY rank the next plan passes (b)
  and (c) against the merged boundary copy -- the non-owner's frozen replica of the winner included, so its planes must
  have been re-split after the broadcast, and a row-sharded winner must have been rebuilt at the full batch -- the
  gathered EMA losses follow the owners, and the frozen replicas, mixture weights and bias are byte-identical."""
  import torch.multiprocessing as mp
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = st._free_port()
  procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, name, fmt, q)) for r in range(2)]
  for p in procs:
    p.start()
  got = {}
  try:
    for _ in procs:
      rank, fails, replicas = q.get(timeout=300)
      got[rank] = (fails, replicas)
  finally:
    for p in procs:
      p.join(timeout=60)
      if p.is_alive():
        p.kill()
        p.join()
  fails = [f for r in sorted(got) for f in got[r][0]]
  assert not fails, "%s:\n%s" % (name, "\n".join(fails[:30]))
  assert all(p.exitcode == 0 for p in procs)
  for t, (a, b) in enumerate(zip(got[0][1], got[1][1])):
    assert len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b)), "after iteration %d the ranks' replicas differ" % t


# ------------------------------------------------------------------------------------------------------------------
# CPU: the float64 initial mixture weights against the oracle's candidates
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mix_type", ["scalar", "vector", "matrix"])
@pytest.mark.parametrize("warm", [False, True])
def test_initial_head_matches_oracle(mix_type, warm):
  """initial_head restates what orc.build_candidates starts a Grow candidate from: 1/N (zeros for MATRIX) for every
  member, or with warm start the previous ensemble's rows for the frozen members and its bias."""
  rng = np.random.default_rng(3)
  C = 10
  frozen_dims = [[D, 32, C], [D, 24, 40, C]]
  frozen = [orc.FrozenMember(0, "f%d" % k, [orc.glorot_uniform(rng, d[i], d[i + 1]) for i in range(len(d) - 1)],
                             [np.zeros(d[i + 1], np.float32) for i in range(len(d) - 1)], 1.0) for k, d in enumerate(frozen_dims)]
  specs = [orc.SubnetworkSpec("n%d" % i, dims, 1.0, ("sgd", 0.1), ws=[orc.glorot_uniform(rng, dims[j], dims[j + 1])
                                                                      for j in range(len(dims) - 1)],
                              bs=[np.zeros(dims[j + 1], np.float32) for j in range(len(dims) - 1)])
           for i, dims in enumerate([[D, 48, C], [D, C]])]
  last = [d[-2] for d in frozen_dims]
  if mix_type == "matrix":
    prev = [rng.standard_normal((d, C)).astype(np.float32) for d in last]
  else:
    prev = rng.uniform(0.1, 0.9, (2,) if mix_type == "scalar" else (2, C)).astype(np.float32)
  prev_b = rng.standard_normal(C).astype(np.float32)
  ens = orc.EnsemblerSpec(optimizer=("sgd", 0.1), mixture_weight_type=mix_type, use_bias=True, warm_start_mixture_weights=warm)
  cands = orc.build_candidates(1, specs, frozen, ens, C, 0.9, prev_weights=prev, prev_bias=prev_b)
  for sp, cs in zip(specs, cands):
    mix, bias = initial_head(mix_type, "complexity_regularized", 2, last + [sp.dims[-2]], C,
                             [prev[k] for k in range(2)] if warm else None, prev_b if warm else None)
    for k, w in enumerate(cs.weights):
      np.testing.assert_array_equal(np.asarray(w, np.float64).reshape(np.shape(mix[k])), mix[k])
    np.testing.assert_array_equal(np.asarray(cs.bias, np.float64), bias)


# ------------------------------------------------------------------------------------------------------------------
# Estimator: the fallback with in-flight checkpoints, and resumes after it
# ------------------------------------------------------------------------------------------------------------------
EB, ED, EC, E_STEPS = 256, 20, 4, 8


def _est_data():
  x, y = orc.make_tabular(EB * 48, ED, EC, seed=4321)
  x = x.copy()
  x[E_STEPS * EB, 3] = SPIKE           # row 0 of iteration 1's first batch
  return x, y


def _estimator(model_dir, save_every):
  import adanet_b200 as adanet
  from adanet_b200 import graph, train
  from adanet_b200.examples import simple_dnn
  from tests.test_gpu_api import SEED, _modern
  gen = _modern(simple_dnn.Generator(feature_columns=[graph.numeric_column("x", ED)],
                                     optimizer=train.MomentumOptimizer(0.02, 0.9), layer_size=16, seed=SEED))
  return adanet.Estimator(
      head=adanet.heads.MultiClassHead(EC), subnetwork_generator=gen, max_iteration_steps=E_STEPS,
      ensemblers=[adanet.ensemble.ComplexityRegularizedEnsembler(optimizer=train.AdamOptimizer(0.01), adanet_lambda=0.01,
                                                                 use_bias=True)],
      max_iterations=3, model_dir=model_dir, config=adanet.RunConfig(model_dir=model_dir, save_checkpoints_steps=save_every),
      debug=True)


def _input_from(x, y, start):
  def fn():
    for i in range(start * EB, x.shape[0] - EB + 1, EB):
      yield {"x": x[i:i + EB]}, y[i:i + EB]
  return fn


def _lib_f16():
  from adanet_b200 import _lib
  return _lib.PLANES_F16


def _fresh_fp16():
  """a new process's plane format"""
  from adanet_b200 import _lib
  _lib.set_plane_format(_lib.PLANES_F16)
  _lib.plane_overflow()


class _Killed(Exception):
  pass


class _KillAfter:
  """a hook that ends the process's training (raises) after n steps"""

  def __init__(self, n):
    self.n = n

  def after_run(self, run_context, run_values):
    self.n -= 1
    if self.n == 0:
      raise _Killed()


def _assert_same_run(got, want, got_dir, want_dir):
  from adanet_b200 import _lib
  assert got._global_step == want._global_step and got._search.iteration == want._search.iteration
  assert got._search.architecture == want._search.architecture
  assert got._search.replay_trace == want._search.replay_trace
  rg, rw = got._search.reports[-1], want._search.reports[-1]
  np.testing.assert_array_equal(rg.ema_losses, rw.ema_losses)
  for nm in rw.traces:
    for f in rw.traces[nm]:
      np.testing.assert_array_equal(rg.traces[nm][f], rw.traces[nm][f], err_msg="%s %s" % (nm, f))
  with np.load(os.path.join(got_dir, "ensemble-latest.npz")) as a, np.load(os.path.join(want_dir, "ensemble-latest.npz")) as b:
    assert sorted(a.files) == sorted(b.files)
    for k in b.files:
      assert _same(a[k], b[k]), "ensemble-latest.npz: %s differs" % k
  with open(os.path.join(got_dir, "ensemble-latest.json")) as f:
    mg = json.load(f)
  with open(os.path.join(want_dir, "ensemble-latest.json")) as f:
    mw = json.load(f)
  assert mg == mw and mw["plane_format"] == "tf32"
  assert _lib.plane_format() == _lib.PLANES_TF32


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", ["inflight_saves", "kill_inside_fp16_attempt", "kill_at_boundary", "kill_inside_rerun"])
def test_estimator_fallback_checkpoints_match_uninterrupted_run(tmp_path, scenario):
  """Iteration 1's first batch overflows fp16; the uninterrupted run without in-flight saves falls back and re-runs
  iteration 1 on TF32 planes over the batches that follow.
    inflight_saves     the same run saving every 3 steps: the re-run must start from the boundary, not from the
                       discarded attempt's in-flight file, and consume the same batches
    kill_at_boundary   killed at the end of the re-run, resumed by a fresh fp16 process: it must continue on TF32
    kill_inside_rerun  killed inside the re-run (in-flight state on TF32 at global step 12), resumed by a fresh fp16
                       process: it must load that state on TF32 planes
    kill_inside_fp16_attempt  killed inside the fp16 attempt after the spike (in-flight state at global step 12):
                       the resumed process must finish the attempt, fall back on the overflow the file carries and
                       re-run the iteration on TF32
  Each ends byte-identical to the uninterrupted run: traces, selections, ensemble-latest.{npz,json}, plane format."""
  from tests.test_gpu_plane_groups import _open
  _open()
  x, y = _est_data()
  full_dir, dir_ = str(tmp_path / "full"), str(tmp_path / scenario)
  _fresh_fp16()
  full = _estimator(full_dir, None)
  full.train(_input_from(x, y, 0), max_steps=3 * E_STEPS)
  assert full._search.tf32_fallbacks == 1
  _fresh_fp16()
  if scenario == "inflight_saves":
    a = _estimator(dir_, 3)
    a.train(_input_from(x, y, 0), max_steps=3 * E_STEPS)
    assert a._search.tf32_fallbacks == 1
    _assert_same_run(a, full, dir_, full_dir)
    return
  # the uninterrupted run consumes 8 + 8 (discarded) + 8 + 8 batches
  a = _estimator(dir_, 3)
  if scenario == "kill_inside_fp16_attempt":
    with pytest.raises(_Killed):
      a.train(_input_from(x, y, 0), hooks=[_KillAfter(E_STEPS + 5)])      # global step 13 of the fp16 attempt
    assert a._global_step == 13 and a._search.plan.fmt == _lib_f16()
    resume_at = E_STEPS + 4              # after the batch of global step 12, the last in-flight save
  elif scenario == "kill_at_boundary":
    a.train(_input_from(x, y, 0), max_steps=2 * E_STEPS)       # global step 16 = the end of the re-run
    assert a._global_step == 2 * E_STEPS and a._search.iteration == 2
    resume_at = 3 * E_STEPS
  else:
    with pytest.raises(_Killed):
      a.train(_input_from(x, y, 0), hooks=[_KillAfter(3 * E_STEPS - 3)])     # global step 13 of the re-run
    assert a._global_step == 13
    resume_at = 2 * E_STEPS + 4          # after the re-run's batch of global step 12, the last in-flight save
  assert getattr(a._search, "tf32_fallbacks", 0) == (0 if scenario == "kill_inside_fp16_attempt" else 1)
  _fresh_fp16()
  b = _estimator(dir_, 3)
  b.train(_input_from(x, y, resume_at), max_steps=3 * E_STEPS)
  _assert_same_run(b, full, dir_, full_dir)
