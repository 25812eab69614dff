"""adanet.Estimator over the B200 engine.

API mirror of adanet/core/estimator.py (`Estimator` :442-2222): constructor
arguments and validation (:604-760), `train` (:809-999), `evaluate`, `predict`,
selection (`_get_best_ensemble_index` :1415-1517) and the per-iteration
`architecture-{t}.json` files (:1408-1413, :1725-1747).  What the reference
does by rebuilding a TF graph 3-4 times per iteration and chaining checkpoints
is a plain Python loop here: per iteration the candidates' builders are called
once against a symbolic graph (core/lowering.py), lowered to a per-GPU
`IterationPlan` (core/engine.py) and stepped with CUDA kernels; selection,
growth and the frozen replay happen in HBM.

Out of scope (SURVEY.md section 2): TensorBoard summaries, report
materialisation, TPU, SavedModel export, parameter-server placement.
"""

from __future__ import annotations

import inspect
import json
import logging
import os
from typing import Dict, List, Optional

import numpy as np

from adanet_b200 import ensemble as ensemble_lib
from adanet_b200 import graph
from adanet_b200 import train as train_lib
from adanet_b200.core import input_utils
from adanet_b200.core.architecture import _Architecture
from adanet_b200.core.metrics import STREAM_METRICS


class RunConfig:
  """The RunConfig fields the estimator reads (tf.estimator.RunConfig stand-in)."""

  def __init__(self, model_dir=None, tf_random_seed=None, num_worker_replicas=None, global_id_in_cluster=None,
               is_chief=None, save_checkpoints_steps=None, **unused):
    ws = int(os.environ.get("WORLD_SIZE", "1"))
    rk = int(os.environ.get("RANK", "0"))
    self.model_dir = model_dir
    self.tf_random_seed = tf_random_seed
    self.num_worker_replicas = num_worker_replicas if num_worker_replicas is not None else ws
    self.global_id_in_cluster = global_id_in_cluster if global_id_in_cluster is not None else rk
    self.num_ps_replicas = 0
    self.save_checkpoints_steps = save_checkpoints_steps   # in-flight iteration state every N global steps
    self.is_chief = is_chief if is_chief is not None else (self.global_id_in_cluster == 0)


class _RunValues:
  """tf.estimator.SessionRunValues stand-in: `.results` holds what the step produced."""

  def __init__(self, results):
    self.results = results


class _Lookahead:
  """Iterator with a one-item peek (the item is handed out by the next `__next__`)."""

  _EMPTY = object()

  def __init__(self, iterable):
    self._it = iter(iterable)
    self._head = self._EMPTY

  def __iter__(self):
    return self

  def __next__(self):
    if self._head is not self._EMPTY:
      item, self._head = self._head, self._EMPTY
      return item
    return next(self._it)

  def peek(self):
    if self._head is self._EMPTY:
      try:
        self._head = next(self._it)
      except StopIteration:
        return None
    return self._head


class _RestoredBuilder:
  """Stands in for the builder of a member restored from a checkpoint (strategies only count / name them)."""

  def __init__(self, name):
    self.name = name


class Estimator(object):
  """An AdaNet estimator: learns an ensemble of subnetworks over iterations.

  Args are those of adanet/core/estimator.py:604-631.  `head` is one of
  adanet_b200.heads.*; `subnetwork_generator` an adanet_b200.subnetwork.Generator
  whose builders use the adanet_b200.graph vocabulary; `ensemblers` defaults to
  one ComplexityRegularizedEnsembler built from the legacy kwargs
  (mixture_weight_type, adanet_lambda, adanet_beta, use_bias,
  warm_start_mixture_weights, mixture_weight_initializer); `ensemble_strategies`
  defaults to [GrowStrategy()].
  """

  def __init__(self, head, subnetwork_generator, max_iteration_steps, ensemblers=None, ensemble_strategies=None,
               evaluator=None, report_materializer=None, metric_fn=None, force_grow=False,
               replicate_ensemble_in_training=False, adanet_loss_decay=.9, delay_secs_per_worker=5,
               max_worker_delay_secs=60, worker_wait_secs=5, worker_wait_timeout_secs=7200, model_dir=None,
               report_dir=None, config=None, debug=False, enable_ensemble_summaries=True,
               enable_subnetwork_summaries=True, global_step_combiner_fn=None, max_iterations=None,
               export_subnetwork_logits=False, export_subnetwork_last_layer=True, replay_config=None, **kwargs):
    if subnetwork_generator is None:
      raise ValueError("subnetwork_generator can't be None.")
    if max_iteration_steps is not None and max_iteration_steps <= 0.:
      raise ValueError("max_iteration_steps must be > 0 or None.")
    if max_iterations is not None and max_iterations <= 0.:
      raise ValueError("max_iterations must be > 0 or None.")
    self._config = config or RunConfig(model_dir=model_dir)
    is_distributed_training = self._config.num_worker_replicas and self._config.num_worker_replicas > 1
    self._model_dir = model_dir or getattr(self._config, "model_dir", None)
    if is_distributed_training and not self._model_dir:
      raise ValueError("For distributed training, a model_dir must be specified.")
    if metric_fn is not None:
      # adanet/core/estimator.py:1718-1760 adds the user's metrics to every candidate's eval metric ops; the engine
      # reports its own fixed set (loss, average_loss, accuracy, ...) -- refusing beats dropping them silently
      raise NotImplementedError("metric_fn (custom evaluation metrics) is not supported by the B200 engine")
    self._replicate_ensemble_in_training = bool(replicate_ensemble_in_training)
    self._head = head
    self._subnetwork_generator = subnetwork_generator
    self._max_iteration_steps = max_iteration_steps
    self._evaluator = evaluator
    self._report_materializer = report_materializer
    self._force_grow = force_grow
    self._adanet_loss_decay = adanet_loss_decay
    self._max_iterations = max_iterations
    self._replay_config = replay_config
    self._debug = debug
    default_ensembler_args = ["mixture_weight_type", "mixture_weight_initializer", "warm_start_mixture_weights",
                              "adanet_lambda", "adanet_beta", "use_bias"]
    default_ensembler_kwargs = {k: v for k, v in kwargs.items() if k in default_ensembler_args}
    if default_ensembler_kwargs:
      logging.warning("The following arguments have been moved to `adanet.ensemble.ComplexityRegularizedEnsembler` "
                      "which can be specified in the `ensemblers` argument: %s", sorted(default_ensembler_kwargs.keys()))
    for key in default_ensembler_kwargs:
      del kwargs[key]
    self._placement_strategy = kwargs.pop("experimental_placement_strategy", None)
    # B200 engine extension: how candidates map to the GPU ranks of a torchrun job -- "balanced" (whole candidates,
    # cost-balanced), "round_robin" (i % G, the reference's RoundRobinStrategy order) or "sharded" (candidates heavier
    # than a rank's share are trained data-parallel over several ranks, distributed/exchange.sharded_placement)
    self._candidate_placement = kwargs.pop("candidate_placement", "balanced")
    if self._candidate_placement == "sharded" and evaluator is not None:
      raise ValueError("candidate_placement='sharded' evaluates candidates on their training shards only; use "
                       "'balanced' together with an Evaluator")
    if default_ensembler_kwargs and ensemblers:
      raise ValueError("When specifying the `ensemblers` argument, the following arguments must not be given: {}".format(
          default_ensembler_kwargs.keys()))
    if not ensemblers:
      if default_ensembler_kwargs.get("warm_start_mixture_weights"):
        default_ensembler_kwargs["model_dir"] = self._model_dir or "."
      ensemblers = [ensemble_lib.ComplexityRegularizedEnsembler(**default_ensembler_kwargs)]
    self._ensemblers = list(ensemblers)
    self._ensemble_strategies = list(ensemble_strategies or [ensemble_lib.GrowStrategy()])
    if self._model_dir:
      os.makedirs(self._model_dir, exist_ok=True)
    # run state
    self._search = None
    self._global_step = 0
    self._iteration_step = 0
    self._batch_size = None
    self._feature_keys = None
    self._in_dim = None
    self._member_subnetworks = []     # Subnetwork namedtuple of every frozen member
    self._member_builders = []
    self._previous_ensemble = None
    self._pending = None              # (builders, subnetworks) of the iteration being trained
    self._eval_plan = None
    self._last_candidate_name = None
    self._architecture = None

  # ------------------------------------------------------------------ properties
  @property
  def model_dir(self):
    return self._model_dir

  @property
  def config(self):
    return self._config

  def latest_checkpoint(self):
    if not self._model_dir:
      return None
    p = os.path.join(self._model_dir, "ensemble-latest.npz")
    return p if os.path.exists(p) else None

  # ------------------------------------------------------------------ engine wiring
  def _ensembler_plan_specs(self):
    """One EnsemblerPlanSpec per `ensemblers` entry: every strategy candidate is built once per ensembler
    (adanet/core/iteration.py:683-693)."""
    return [self._ensembler_plan_spec(e) for e in self._ensemblers]

  def _ensembler_plan_spec(self, e=None):
    from adanet_b200.core import engine as eng
    e = e if e is not None else self._ensemblers[0]
    # The engine runs the arithmetic of the two built-in ensemblers in its own kernels.  A subclass may rename or
    # re-parameterise them, but one that overrides the arithmetic itself would be silently ignored: refuse it.
    for base in (ensemble_lib.MeanEnsembler, ensemble_lib.ComplexityRegularizedEnsembler):
      if isinstance(e, base):
        for meth in ("build_ensemble", "build_train_op", "complexity_regularization", "_compute_adanet_gamma"):
          if hasattr(base, meth) and getattr(type(e), meth) is not getattr(base, meth):
            raise NotImplementedError("custom Ensemblers are not supported by the B200 engine: %s overrides %s.%s"
                                      % (type(e).__name__, base.__name__, meth))
    if isinstance(e, ensemble_lib.MeanEnsembler):
      # mean over the candidate's NEW subnetworks only (adanet/ensemble/mean.py:92-101; previous members are
      # ignored, nothing is trained): SCALAR weights 0 for kept members, 1/n_new for the new ones
      return eng.EnsemblerPlanSpec(optimizer=None, mixture_weight_type="scalar", name=e.name, kind="mean")
    if not isinstance(e, ensemble_lib.ComplexityRegularizedEnsembler):
      raise NotImplementedError("custom Ensemblers are not supported by the B200 engine: %r" % (e,))
    return eng.EnsemblerPlanSpec(optimizer=train_lib.optimizer_from(e.optimizer), mixture_weight_type=e.mixture_weight_type,
                                 adanet_lambda=e.adanet_lambda, adanet_beta=e.adanet_beta, use_bias=e.use_bias,
                                 name=e.name, warm_start_mixture_weights=bool(e.warm_start_mixture_weights),
                                 initial_weight_fn=(e.initial_mixture_weight
                                                    if getattr(e, "_mixture_weight_initializer", None) is not None else None))

  def _check_strategies(self):
    for s in self._ensemble_strategies:
      if not isinstance(s, ensemble_lib.Strategy):
        raise ValueError("ensemble_strategies must be adanet.ensemble.Strategy instances, got %r" % (s,))

  def _generate_builders(self, iteration_number):
    gen = self._subnetwork_generator
    kwargs = dict(previous_ensemble=self._previous_ensemble, iteration_number=iteration_number,
                  previous_ensemble_reports=[], all_reports=[])
    if "config" in inspect.signature(gen.generate_candidates).parameters:
      kwargs["config"] = self._config
    builders = list(gen.generate_candidates(**kwargs))
    if not builders:
      raise ValueError("Each iteration must have at least one Builder.")
    return builders

  def _search_space(self, iteration_number, frozen):
    """Generator -> Strategy -> Builder.build_subnetwork -> lowering, for iteration t
    (adanet/core/estimator.py:2107-2117 + iteration.py:628-652)."""
    from adanet_b200.core import lowering
    builders = self._generate_builders(iteration_number)
    names = [b.name for b in builders]
    for n in names:
      if names.count(n) > 1:
        raise ValueError("Two subnetworks have the same name '{}'".format(n))
    from adanet_b200.core import search as srch
    cands = []
    for strategy in self._ensemble_strategies:
      cands += list(strategy.generate_ensemble_candidates(builders, list(self._member_builders)))
    ecands = []
    for c in cands:     # strategy.py:26-76: (name, new builders, previous builders kept | None)
      prev = c.previous_ensemble_subnetwork_builders
      # ensemble_builder.py:367-388: previous members are kept, in order, when their builder is among the candidate's
      # previous_ensemble_subnetwork_builders (and survives a single builder's deprecated prune_previous_ensemble)
      keep = [i for i, b in enumerate(self._member_builders) if prev and b in prev]
      if len(c.subnetwork_builders) == 1 and self._previous_ensemble is not None:
        legacy = getattr(c.subnetwork_builders[0], "prune_previous_ensemble", None)
        if callable(legacy):
          logging.warning("Using an `adanet.subnetwork.Builder#prune_previous_ensemble` is deprecated. Please use a "
                          "custom `adanet.ensemble.Strategy` instead.")
          allowed = set(int(i) for i in legacy(self._previous_ensemble))
          keep = [i for i in keep if i in allowed]
      keeps = True if (len(keep) == len(self._member_builders)) else (keep if keep else False)
      ecands.append(srch.EnsembleCandidate(c.name, [builders.index(b) for b in c.subnetwork_builders], keeps))
    self._pending_ecands = ecands
    # image features keep their [batch, H, W, C] shape for the builder; everything else is [batch, width]
    placeholders = {k: graph.placeholder(self._feature_shapes[k] if len(self._feature_shapes.get(k, ())) == 3 else w, k)
                    for k, w in self._feature_widths.items()}
    labels_ph = graph.placeholder(1, "labels")
    specs, subs = [], []
    for b in builders:
      spec, sub = lowering.build_and_lower(b, placeholders, labels_ph, self._head, iteration_step=0,
                                           previous_ensemble=self._previous_ensemble, in_dim=self._in_dim,
                                           config=self._config, iteration=iteration_number)
      specs.append(spec)
      subs.append(sub)
    if self._replicate_ensemble_in_training and any(sp.dropout and any(d is not None for d in sp.dropout) for sp in specs):
      # the engine replays frozen members in inference mode (the reference's default, ensemble_builder.py:367-388 with
      # replicate_ensemble_in_training=False); with dropout in the search space TRAIN-mode replay would differ
      raise NotImplementedError("replicate_ensemble_in_training=True with dropout in the search space: frozen members "
                                "are replayed without dropout by the B200 engine")
    self._pending = (builders, subs)
    # bagged candidates: a fresh iterator over their own train_input_fn for this iteration (the reference builds a
    # new one-shot iterator with every iteration graph, autoensemble/common.py:151-160)
    self._bagging_iters = {i: iter(input_utils.iterate_input_fn(b.bagging_train_input_fn))
                           for i, (b, sp) in enumerate(zip(builders, specs)) if sp.own_input}
    self._apply_legacy_mixture_weights_train_op(builders, subs, labels_ph)
    return specs

  def _next_bagging_batches(self):
    """One minibatch per bagged candidate for the coming step; None when any of them ran out of data (the
    reference's OutOfRangeError ends training, autoensemble/common.py:75-78)."""
    out = {}
    for i, it in getattr(self, "_bagging_iters", {}).items():
      try:
        f, l = next(it)
      except StopIteration:
        logging.info("bagging input of candidate %d is exhausted: training stops", i)
        return None
      if input_utils.batch_size_of(f) != self._batch_size:
        raise ValueError("bagging train_input_fn of candidate %d yields batches of %d examples, the Estimator's input_fn %d"
                         % (i, input_utils.batch_size_of(f), self._batch_size))
      out[i] = (input_utils.to_matrix(f, self._feature_keys), l)
    return out

  def _apply_legacy_mixture_weights_train_op(self, builders, subs, labels_ph):
    """adanet/core/ensemble_builder.py:523-537: a candidate whose first builder still defines the deprecated
    `build_mixture_weights_train_op` trains its mixture weights with THAT op (given loss=adanet_loss, so the
    regulariser is counted once), not with `Ensembler.build_train_op`.  The engine runs one mixture-weight
    optimizer per iteration, so all builders of an iteration must agree."""
    import dataclasses
    from adanet_b200 import train
    from adanet_b200.core import lowering
    fns = [getattr(b, "build_mixture_weights_train_op", None) for b in builders]
    if self._search is None:
      return
    if len(self._ensemblers) > 1:
      if any(callable(f) for f in fns):
        raise NotImplementedError("the deprecated build_mixture_weights_train_op with several ensemblers is not "
                                  "implemented by the B200 engine")
      return
    base = self._ensembler_plan_spec()
    if not any(callable(f) for f in fns) or base.kind == "mean":
      self._search.ens = base
      return
    if not all(callable(f) for f in fns):
      raise NotImplementedError("builders with and without the deprecated build_mixture_weights_train_op in one "
                                "iteration are not implemented by the B200 engine")
    logging.warning("The `build_mixture_weights_train_op` method is deprecated. Please use the `Ensembler#build_train_op` instead.")
    specs = set()
    for b, f, sub in zip(builders, fns, subs):
      op = f(loss=self._head.create_loss(sub.logits), var_list=[], logits=sub.logits, labels=labels_ph, iteration_step=0,
             summary=lowering._NullSummary())
      op = op.train_op if hasattr(op, "train_op") and not isinstance(op, train.TrainOp) else op
      if not isinstance(op, train.TrainOp):
        raise ValueError("build_mixture_weights_train_op of %s must return optimizer.minimize(...) or tf.no_op(), got %r" % (b.name, op))
      specs.add(None if op.kind == "no_op" else tuple(op.spec))
    if len(specs) != 1:
      raise NotImplementedError("builders whose build_mixture_weights_train_op differ within one iteration are not implemented")
    self._search.ens = dataclasses.replace(base, optimizer=specs.pop(), legacy_train_op=True)

  def _ensure_search(self, features):
    from adanet_b200.core import search as srch
    if self._search is not None:
      return
    self._check_strategies()
    self._batch_size = input_utils.batch_size_of(features)
    widths = input_utils.feature_widths(features)
    self._feature_keys = sorted(widths)
    self._feature_widths = widths
    self._feature_shapes = input_utils.feature_shapes(features)
    self._in_dim = sum(widths.values())
    replay = self._replay_config.best_ensemble_indices if self._replay_config else None
    self._search = srch.AdaNetSearch(self._search_space, self._ensembler_plan_specs(), self._in_dim,
                                     self._head.logits_dimension, self._batch_size, head=self._head.loss_kind,
                                     adanet_loss_decay=self._adanet_loss_decay, force_grow=self._force_grow,
                                     replay_indices=replay, keep_traces=bool(self._debug),
                                     candidates_fn=lambda specs, n_frozen: self._pending_ecands,
                                     placement=self._candidate_placement)

  def _inflight_path(self):
    return os.path.join(self._model_dir, "iteration-inflight-rank{}.npz".format(self._config.global_id_in_cluster))

  def _save_inflight(self):
    """Mid-iteration checkpoint (every `RunConfig.save_checkpoints_steps` global steps): the candidates' weights,
    optimizer slots, mixture weights, EMA and step counters of THIS rank's shard, so a killed run resumes
    inside the iteration (the reference persists the same through the TF checkpoint,
    adanet/core/iteration.py:40-118,172-183).  Candidate builders are re-generated deterministically on resume."""
    st = self._search.plan.state_dict()
    st["meta_plane_format"] = np.asarray(self._search.plan.fmt, dtype=np.int64)
    # the sticky overflow flag, read without clearing it: a run resumed from here must fall back as this one will
    st["meta_plane_overflow"] = np.asarray(self._search.plan.plane_overflow(reset=False), dtype=np.int64)
    st["meta_iteration"] = np.asarray(self._search.iteration, dtype=np.int64)
    st["meta_global_step"] = np.asarray(self._global_step, dtype=np.int64)
    st["meta_iteration_step"] = np.asarray(self._iteration_step, dtype=np.int64)
    tmp = self._inflight_path() + ".tmp.npz"
    np.savez(tmp, **st)
    os.replace(tmp, self._inflight_path())

  def _maybe_restore_inflight(self):
    """Called right after an iteration's plan was built: loads the in-flight state if it belongs to it.

    The state belongs to it when it was saved in this iteration, at or after the current global step, on the plan's
    plane format.  A file on TF32 planes while the plan is on fp16 ones was written by a run that fell back inside this
    iteration (core/search.py restart_on_tf32_if_overflowed): this process falls back too and rebuilds the plan before
    loading it.  A file on fp16 planes while the plan is on TF32 ones is a discarded attempt and is refused."""
    if not self._model_dir or self._iteration_step != 0:
      return False
    from adanet_b200 import _lib
    from adanet_b200.distributed import exchange as ex
    plan = self._search.plan
    st, ok = None, False
    if os.path.exists(self._inflight_path()):
      st = dict(np.load(self._inflight_path()))
      ok = int(st["meta_iteration"]) == self._search.iteration and int(st["meta_global_step"]) >= self._global_step
      if ok and plan.xp is not None and self._inflight_format(st) != plan.fmt:
        ok = self._inflight_format(st) == _lib.PLANES_TF32
    # every rank resumes from the same global step or none does (ranks killed at different save points would otherwise
    # reach the end-of-iteration collectives at different times); all ranks take part in the agreement, file or not
    mine = float(st["meta_global_step"]) if ok else -1.0
    lo = -ex.max_over_ranks(-mine, device=self._search.device)
    hi = ex.max_over_ranks(mine, device=self._search.device)
    if lo != hi or lo < 0:
      if ok:
        logging.warning("in-flight checkpoints of the ranks disagree (steps %s..%s): restarting iteration %d", lo, hi,
                        self._search.iteration)
      return False
    if plan.xp is not None and self._inflight_format(st) != plan.fmt:
      # every rank saved this step on the same format (the fallback is agreed by all_reduce), so all of them get here
      logging.warning("iteration %d: the in-flight checkpoint was written on TF32 planes after an fp16 overflow; "
                      "continuing on TF32 planes", self._search.iteration)
      _lib.set_plane_format(_lib.PLANES_TF32)
      self._search.build_iteration()
    self._search.plan.load_state_dict(st)
    self._search.plan.carried_overflow = bool(int(st.get("meta_plane_overflow", 0)))
    self._global_step = int(st["meta_global_step"])
    self._iteration_step = int(st["meta_iteration_step"])
    for it in getattr(self, "_bagging_iters", {}).values():      # bagging inputs restart with the iteration: skip what it consumed
      for _ in range(self._iteration_step):
        next(it, None)
    logging.info("resumed iteration %d at iteration step %d (global step %d)", self._search.iteration,
                 self._iteration_step, self._global_step)
    return True

  @staticmethod
  def _inflight_format(st):
    """Plane format an in-flight state was saved on; files written before it was recorded were on fp16 planes."""
    from adanet_b200 import _lib
    return int(st["meta_plane_format"]) if "meta_plane_format" in st else _lib.PLANES_F16

  def _maybe_restore(self):
    """Continues from `model_dir/ensemble-latest.{npz,json}` (written at every iteration boundary): frozen
    members, mixture weights, selection state and step counters -- what the reference restores from
    `increment.ckpt-{t}` + `architecture-{t}.json` when an Estimator is re-created on the same model_dir
    (adanet/core/estimator.py:951-984)."""
    from adanet_b200 import subnetwork as subnetwork_lib
    from adanet_b200.core import engine as eng
    path = self.latest_checkpoint()
    meta_path = os.path.join(self._model_dir, "ensemble-latest.json") if self._model_dir else None
    if not path or not meta_path or not os.path.exists(meta_path) or self._search.iteration > 0:
      return False
    with open(meta_path) as f:
      meta = json.load(f)
    if int(meta["batch_size"]) != int(self._batch_size) or {k: int(v) for k, v in meta["feature_widths"].items()} != \
        {k: int(v) for k, v in self._feature_widths.items()}:
      raise ValueError("model_dir %s holds a checkpoint for batch size %s / features %s, input_fn yields %s / %s" % (
          self._model_dir, meta["batch_size"], meta["feature_widths"], self._batch_size, self._feature_widths))
    data = np.load(path)
    if int(data["iteration"]) != int(meta["iteration"]) or int(data["global_step"]) != int(meta["global_step"]):
      raise ValueError("model_dir %s: ensemble-latest.npz (iteration %d, step %d) and ensemble-latest.json (iteration %d, "
                       "step %d) belong to different checkpoints" % (self._model_dir, int(data["iteration"]),
                                                                     int(data["global_step"]), int(meta["iteration"]),
                                                                     int(meta["global_step"])))
    s = self._search
    if meta.get("plane_format") == "tf32":
      # the run that wrote it fell back from fp16 planes (core/search.py restart_on_tf32_if_overflowed), which is for
      # good: continue on TF32 as it did.  A checkpoint on fp16 planes, or one written before the format was recorded,
      # leaves the process's format alone.
      from adanet_b200 import _lib
      if _lib.plane_format() != _lib.PLANES_TF32:
        logging.info("model_dir %s was trained on TF32 planes: switching to them", self._model_dir)
        _lib.set_plane_format(_lib.PLANES_TF32)
    from adanet_b200.core import lowering
    dims_of = {(int(m["iteration"]), m["name"]): m["dims"] for m in meta["members"]}
    dims_of = lambda it, name, _d=dims_of: _d[(int(it), name)]
    members = []
    for k, m in enumerate(meta["members"]):
      n_layers = len(m["dims"]) - 1 + (1 if m.get("image_shape") else 0)     # a conv stem's kernel / bias come first
      ws = [data["m{}_w{}".format(k, i)] for i in range(n_layers)]
      bs = [data["m{}_b{}".format(k, i)] for i in range(n_layers)]
      # a member reads only members before it (the order the ensemble grew in)
      members.append(eng.DenseNet(m["name"], m["dims"], ws, bs, m["complexity"], s.batch, s.device, m["iteration"],
                                  lowering.decode_tensors(m["shared"], dims_of, s.in_dim), m.get("image_shape"),
                                  inputs=m.get("inputs"), members=list(members)))
    s.frozen = members
    s.iteration = int(meta["iteration"])
    s.architecture = [(int(t), n) for t, n in meta["architecture"]]
    s.replay_trace = list(meta["replay_trace"])
    s.prev_best_ema = meta["prev_best_ema"]
    if "mixture_weights" in data:
      s.mixture_weights = data["mixture_weights"]
    else:
      s.mixture_weights = [data["mixture_weight_{}".format(k)] for k in range(len(members))]
    s.bias = data["bias"]
    self._global_step = int(meta["global_step"])
    self._last_candidate_name = meta["last_candidate_name"]
    # previous_ensemble for the generator: symbolic subnetworks carrying complexity + shared (what builders read)
    s.winner_ens_index = int(meta.get("winner_ens_index", 0))
    ens = self._ensemblers[s.winner_ens_index]
    self._member_subnetworks, self._member_builders, ws_list = [], [], []
    mw = s.mixture_weights
    for k, m in enumerate(meta["members"]):
      sub = lowering.restored_subnetwork(m, dims_of, s.in_dim)
      lg = sub.logits
      self._member_subnetworks.append(sub)
      self._member_builders.append(_RestoredBuilder(m["name"]))
      ws_list.append(ensemble_lib.WeightedSubnetwork(name=m["name"], iteration_number=m["iteration"],
                                                     weight=np.array(mw[k]), logits=lg, subnetwork=sub))
    self._previous_ensemble = ensemble_lib.ComplexityRegularized(
        weighted_subnetworks=ws_list, bias=np.asarray(s.bias), logits=("weighted_sum", [w.logits for w in ws_list]),
        subnetworks=[w.subnetwork for w in ws_list],
        complexity_regularization=ens.complexity_regularization([w.weight for w in ws_list],
                                                                [w.subnetwork.complexity for w in ws_list]))
    arch = _Architecture(self._last_candidate_name, ens.name, replay_indices=list(s.replay_trace))
    for t, n in s.architecture:
      arch.add_subnetwork(t, n)
    self._architecture = arch
    logging.info("restored iteration %d (global step %d) from %s", s.iteration, self._global_step, path)
    return True

  # ------------------------------------------------------------------ train
  def train(self, input_fn, hooks=None, steps=None, max_steps=None, saving_listeners=None):
    """Trains for `steps` more steps or until `max_steps` global steps
    (adanet/core/estimator.py:809-999).  An AdaNet iteration ends after
    `max_iteration_steps` steps (or when the input is exhausted); the best
    candidate is then selected and frozen, and the next iteration starts.

    `hooks`: objects with the SessionRunHook method `after_run(run_context, run_values)`; after every step it is
    called with `run_values.results = {"global_step": int, "losses": float32[n_candidates, 4]}` (sub_loss, ens_loss,
    adanet_loss, ema of this rank's candidate ensembles, read back from the device -- which synchronises on the
    step, so pass hooks only when per-step values are wanted; `begin()` / `end(session)` are called if present."""
    hooks = list(hooks or [])
    for h in hooks:
      if hasattr(h, "begin"):
        h.begin()
    try:
      return self._train(input_fn, hooks, steps, max_steps)
    finally:
      for h in hooks:
        if hasattr(h, "end"):
          h.end(None)

  def _train(self, input_fn, hooks, steps, max_steps):
    if steps is not None and max_steps is not None:
      raise ValueError("Can not provide both steps and max_steps.")
    if steps is not None and steps <= 0:
      raise ValueError("Must specify steps > 0, given: {}".format(steps))
    if max_steps is not None and max_steps <= 0:
      raise ValueError("Must specify max_steps > 0, given: {}".format(max_steps))
    limit = None
    if steps is not None:
      limit = self._global_step + steps
    if max_steps is not None:
      limit = max_steps
      if self._global_step >= max_steps:
        logging.info("Skipping training since max_steps has already saved.")
        return self
    done_iterations = lambda: self._search.iteration if self._search else 0
    # The reference calls `input_fn` anew for every iteration (temp_estimator.train(input_fn=...) inside the loop of
    # adanet/core/estimator.py:890-897): a finite input therefore ends an ITERATION, not training.  Here one pass over
    # the input may span several iterations (max_iteration_steps); when it runs out the iteration in flight is
    # closed and, if max_steps / max_iterations still allow, the input is re-created for the next one.
    while True:
      steps_before = self._global_step
      exhausted = self._train_pass(input_fn, hooks, steps, limit_box := [limit])
      limit = limit_box[0]
      if not exhausted or self._global_step == steps_before:
        break
      if (self._max_iterations and done_iterations() >= self._max_iterations) or (
          limit is not None and self._global_step >= limit):
        break
      if limit is None and not self._max_iterations:
        break      # nothing bounds training: one pass over the input (the reference would loop until interrupted)
    return self

  def _train_pass(self, input_fn, hooks, steps, limit_box):
    """One pass over `input_fn`; returns True when the input ran out (False: a limit stopped training first)."""
    limit = limit_box[0]
    done_iterations = lambda: self._search.iteration if self._search else 0
    batches = _Lookahead(input_utils.iterate_input_fn(input_fn))
    staged = None        # (item, plan) whose host->device copy was started while the previous step ran
    for item in batches:
      features, labels = item
      if self._max_iterations and done_iterations() >= self._max_iterations:
        return False
      if limit is not None and self._global_step >= limit:
        return False
      if self._search is None:
        self._ensure_search(features)
        if self._maybe_restore() and steps is not None:
          limit = limit_box[0] = self._global_step + steps        # `steps` counts from the restored global step
        if (self._max_iterations and done_iterations() >= self._max_iterations) or (
            limit is not None and self._global_step >= limit):
          return False
      bs = input_utils.batch_size_of(features)
      if bs != self._batch_size:
        input_utils.warn_ragged(bs, self._batch_size)
        continue
      if self._search.plan is None:
        self._search.build_iteration()
        self._iteration_step = 0
        if self._maybe_restore_inflight() and steps is not None:
          limit = limit_box[0] = self._global_step + steps
      x = input_utils.to_matrix(features, self._feature_keys)
      own = self._next_bagging_batches()
      if own is None:
        return False
      plan = self._search.plan
      if staged is not None and staged[0] is item and staged[1] is plan:
        plan.train_step(own_batches=own or None)          # the minibatch is already on the device
      else:
        plan.train_step(x, labels, own_batches=own or None)
      staged = None
      self._global_step += 1
      self._iteration_step += 1
      ends_iteration = self._max_iteration_steps is not None and self._iteration_step >= self._max_iteration_steps
      if not ends_iteration and (limit is None or self._global_step < limit):
        # the step above only ENQUEUED work: start the next minibatch's host->device copy on the copy stream now, so
        # it runs under this step's kernels (pageable NumPy input blocks the host for the copy, not the GPU)
        nxt = batches.peek()
        if nxt is not None and input_utils.batch_size_of(nxt[0]) == self._batch_size:
          plan.stage_batch(input_utils.to_matrix(nxt[0], self._feature_keys), nxt[1])
          staged = (nxt, plan)
      if hooks:      # after the next copy was started: reading the losses back waits for the step to finish
        values = _RunValues({"global_step": self._global_step, "losses": plan.last_losses()})
        for h in hooks:
          h.after_run(None, values)
      if ends_iteration:
        self._bookkeeping()
      else:
        every = getattr(self._config, "save_checkpoints_steps", None)
        if every and self._model_dir and self._global_step % int(every) == 0:
          self._save_inflight()
    # input exhausted: the iteration is over (iteration.py:274-284 stops each spec on OutOfRangeError)
    if self._search is not None and self._search.plan is not None and self._iteration_step > 0 and (
        limit is None or self._global_step < limit):
      self._bookkeeping()
    return True

  def _bookkeeping(self):
    """_execute_bookkeeping_phase (estimator.py:1247-1283): evaluate candidates, pick the best,
    write architecture-{t}.json, grow."""
    s = self._search
    t = s.iteration
    if s.restart_on_tf32_if_overflowed():
      # the iteration is trained again (TF32 planes) on the input that follows; its steps do not count, and neither
      # does what the discarded attempt saved in flight (every rank falls back here together and drops its own file)
      self._global_step -= self._iteration_step
      self._iteration_step = 0
      if self._model_dir and os.path.exists(self._inflight_path()):
        os.remove(self._inflight_path())
      return None
    builders, subs = self._pending
    if self._evaluator is not None and self._evaluator.metric_name in STREAM_METRICS:
      ev, name = self._evaluator, self._evaluator.metric_name
      to_x = lambda f: input_utils.to_matrix(f, self._feature_keys)
      prev_metric = None
      if t > 0:
        plan_prev = self._ensemble_eval_plan()
        acc = plan_prev.stream_metrics(name)
        prev_metric = ev.evaluate_streaming(lambda f, l: plan_prev.stream_eval_step(to_x(f), l),
                                            lambda: acc.values(name))[0]
      def local_metric(plan):
        acc = plan.stream_metrics(name)
        return ev.evaluate_streaming(lambda f, l: plan.stream_eval_step(to_x(f), l), lambda: acc.values(name))
      rep = s.finish_iteration(local_metric_fn=local_metric, previous_metric=prev_metric, objective_fn=ev.objective_fn)
    elif self._evaluator is not None:
      ev = self._evaluator
      prev_metric = None
      if t > 0:
        plan_prev = self._ensemble_eval_plan()
        prev_metric = ev.evaluate(lambda f, l: [plan_prev.metric(input_utils.to_matrix(f, self._feature_keys), l,
                                                                 ev.metric_name)], 1)[0]
      def local_metric(plan):
        # the metric the Evaluator names, of every candidate ensemble (estimator.py:1483-1490)
        return ev.evaluate(lambda f, l: plan.eval_step(input_utils.to_matrix(f, self._feature_keys), l, ev.metric_name),
                           len(plan.heads))
      rep = s.finish_iteration(local_metric_fn=local_metric, previous_metric=prev_metric, objective_fn=ev.objective_fn)
    else:
      rep = s.finish_iteration()
    ens = self._ensemblers[s.winner_ens_index]        # the ensembler that built the (new or kept) best ensemble
    if s.last_winner_builders is not None:
      # e.g. SoloStrategy drops the previous ensemble's subnetworks, a pruning Strategy keeps some of them
      kept = getattr(s, "last_winner_kept", None)
      if kept is not None and len(kept) != len(self._member_subnetworks):
        self._member_subnetworks = [self._member_subnetworks[i] for i in kept]
        self._member_builders = [self._member_builders[i] for i in kept]
      for ci in s.last_winner_builders:
        self._member_subnetworks.append(subs[ci])
        self._member_builders.append(builders[ci])
      cand_name = s.last_winner_name
    else:
      cand_name = self._last_candidate_name
    self._last_candidate_name = cand_name
    # previous_ensemble handed to the generator / builders of iteration t+1 (weighted.py:90-136)
    ws = []
    mw = rep.mixture_weights if isinstance(rep.mixture_weights, list) else np.asarray(rep.mixture_weights)
    for k, (sub, (it, name)) in enumerate(zip(self._member_subnetworks, rep.architecture)):
      ws.append(ensemble_lib.WeightedSubnetwork(name=name, iteration_number=it, weight=np.array(mw[k]), logits=sub.logits,
                                                subnetwork=sub))
    if isinstance(ens, ensemble_lib.MeanEnsembler):
      # mean.py:92-135: a MeanEnsemble carries the candidate's new subnetworks only
      n_new = len(s.last_winner_builders) if s.last_winner_builders is not None else len(self._previous_ensemble.subnetworks)
      new_subs = self._member_subnetworks[-n_new:]
      self._previous_ensemble = ensemble_lib.MeanEnsemble(logits=("mean", [sb.logits for sb in new_subs]),
                                                          subnetworks=new_subs, predictions=None)
    else:
      self._previous_ensemble = ensemble_lib.ComplexityRegularized(
          weighted_subnetworks=ws, bias=np.asarray(rep.bias), logits=("weighted_sum", [w.logits for w in ws]),
          subnetworks=[w.subnetwork for w in ws],
          complexity_regularization=ens.complexity_regularization([w.weight for w in ws],
                                                                  [w.subnetwork.complexity for w in ws]))
    arch = _Architecture(cand_name, ens.name, replay_indices=list(rep.replay_indices))
    for it, name in rep.architecture:
      arch.add_subnetwork(it, name)
    self._architecture = arch
    self._eval_plan = None
    self._iteration_step = 0
    if self._model_dir and self._config.is_chief:
      with open(os.path.join(self._model_dir, "architecture-{}.json".format(t)), "w") as f:
        f.write(arch.serialize(t, self._global_step))
      self._save_ensemble()
    logging.info("iteration %d: best ensemble '%s' (index %d)", t, rep.candidate_names[rep.best_index], rep.best_index)
    return rep

  def _save_ensemble(self):
    """The final ensemble's parameters (replaces the reference's increment.ckpt-{t})."""
    from adanet_b200 import _lib
    s = self._search
    fmt = _lib.plane_format()
    out = {"global_step": self._global_step, "iteration": s.iteration, "bias": s.bias, "plane_format": fmt}
    if isinstance(s.mixture_weights, list):
      for k, w in enumerate(s.mixture_weights):
        out["mixture_weight_{}".format(k)] = w
    else:
      out["mixture_weights"] = s.mixture_weights
    from adanet_b200.core import lowering
    for k, m in enumerate(s.frozen):
      ws, bs = m.numpy_params()
      for i, (w, b) in enumerate(zip(ws, bs)):
        out["m{}_w{}".format(k, i)] = w
        out["m{}_b{}".format(k, i)] = b
    # written to a temporary file and renamed, BEFORE the json that points at it; both carry (iteration, global_step)
    # and _maybe_restore refuses a pair that disagrees (a crash between the two renames)
    tmp_npz = os.path.join(self._model_dir, "ensemble-latest.tmp.npz")
    np.savez(tmp_npz, **out)
    os.replace(tmp_npz, os.path.join(self._model_dir, "ensemble-latest.npz"))
    # everything else a fresh process needs to continue from this iteration boundary (the reference keeps it in
    # the TF checkpoint + architecture-{t}.json, adanet/core/estimator.py:1357-1413)
    meta = {
        "global_step": int(self._global_step), "iteration": int(s.iteration),
        "batch_size": int(self._batch_size), "feature_widths": self._feature_widths,
        "architecture": [[int(t), n] for t, n in s.architecture], "replay_trace": [int(v) for v in s.replay_trace],
        "prev_best_ema": None if s.prev_best_ema is None else float(s.prev_best_ema),
        "last_candidate_name": self._last_candidate_name, "winner_ens_index": int(s.winner_ens_index),
        "plane_format": "tf32" if fmt == _lib.PLANES_TF32 else "fp16",
        "members": [self._member_record(k, m, lowering) for k, m in enumerate(s.frozen)],
    }
    tmp = os.path.join(self._model_dir, "ensemble-latest.json.tmp")
    with open(tmp, "w") as f:
      json.dump(meta, f)
    os.replace(tmp, os.path.join(self._model_dir, "ensemble-latest.json"))

  def _member_record(self, k, m, lowering):
    """A frozen member's entry in ensemble-latest.json.  Tensors in `shared` are saved as references to the layers
    they are (lowering.encode_tensors); a member over a concat adds its pieces ("inputs"), and one whose
    persisted_tensors hold tensors adds those."""
    rec = {"name": m.name, "iteration": int(m.iteration), "complexity": float(m.complexity),
           "dims": [int(d) for d in m.dims], "shared": lowering.encode_tensors(m.shared),
           "image_shape": list(m.image_shape) if m.stem else None}
    if m.inputs is not None:
      rec["inputs"] = m.inputs
    subs = getattr(self, "_member_subnetworks", None) or []
    pt = subs[k].persisted_tensors if k < len(subs) else None
    if pt and lowering.encode_tensors(pt) is not pt:
      rec["persisted_tensors"] = lowering.encode_tensors(pt)
    return rec

  # ------------------------------------------------------------------ evaluate / predict
  def _restore_for_inference(self, input_fn):
    """evaluate / predict on a fresh Estimator whose model_dir holds a trained ensemble: shapes come from the
    first batch of `input_fn`, the ensemble from the latest checkpoint (the reference rebuilds the graph from
    architecture-{t}.json and restores increment.ckpt-{t}, adanet/core/estimator.py:1785-1882)."""
    if self._search is not None or not self._model_dir or not self.latest_checkpoint():
      return
    for item in input_utils.iterate_input_fn(input_fn):
      self._ensure_search(item[0] if isinstance(item, tuple) else item)
      self._maybe_restore()
      return

  def _ensemble_eval_plan(self):
    from adanet_b200.core import engine as eng
    s = self._search
    if s is None or not s.frozen:
      raise ValueError("no trained ensemble yet: train at least one AdaNet iteration before evaluate/predict")
    from adanet_b200 import _lib
    if self._eval_plan is None or self._eval_plan.fmt != _lib.plane_format():
      # built anew after the fp16 -> TF32 fallback too: its planes (and the members', EnsembleEvalPlan re-creates
      # them) are sized by the format they were built in
      self._eval_plan = eng.EnsembleEvalPlan(s.frozen, s.mixture_weights, s.bias, s.winner_ens, s.head, s.batch, s.C, s.device)
    return self._eval_plan

  def architecture_string(self):
    """`architecture/adanet/ensembles` text (adanet/core/eval_metrics.py:243-244)."""
    return "| {} |".format(" | ".join(name for _, name in self._architecture.subnetworks))

  def evaluate(self, input_fn, steps=None, hooks=None, checkpoint_path=None, name=None):
    """Metrics of the best ensemble over `steps` batches of at most the training batch size, a partial last batch
    included: `loss` (the mean of the per-batch mean losses), `average_loss` (the mean over examples), `accuracy`
    for classification heads (over examples), `global_step`, `iteration` and the architecture string
    (eval_metrics.py:120,227-264,347-393); a BinaryClassHead adds `precision`, `recall`, `auc`,
    `auc_precision_recall`, `prediction/mean`, `label/mean` and `accuracy_baseline`, a RegressionHead
    `prediction/mean` and `label/mean` (the v2 heads' metrics, streamed over every batch: core/metrics.py)."""
    import torch
    from adanet_b200.core import engine as eng
    self._restore_for_inference(input_fn)
    plan = self._ensemble_eval_plan()
    streams = self._head.loss_kind in ("sigmoid_xent", "mse")
    acc = plan.stream_metrics() if streams else None
    n, loss_sum, examples, example_loss_sum, correct, total = 0, 0.0, 0, 0.0, 0, 0
    for features, labels in input_utils.iterate_input_fn(input_fn):
      if steps is not None and n >= steps:
        break
      loss, _, _ = plan.run(input_utils.to_matrix(features, self._feature_keys), labels)
      b = plan.rows
      loss_sum += loss
      n += 1
      example_loss_sum += loss * b
      examples += b
      if streams:
        plan.add_metrics()
      if self._head.loss_kind != "mse":
        c, t = eng.correct_of(plan.ens_logits[:b], torch.as_tensor(labels).to(plan.device))
        correct += c
        total += t
    if n == 0:
      raise ValueError("evaluate: input_fn produced no batches")
    out = {"loss": loss_sum / n, "average_loss": example_loss_sum / examples, "global_step": self._global_step,
           "iteration": self._search.iteration, "architecture/adanet/ensembles": self.architecture_string()}
    if total:
      out["accuracy"] = correct / total
    if streams:
      out.update(acc.results()[0])
    return out

  def predict(self, input_fn, predict_keys=None, hooks=None, checkpoint_path=None, yield_single_examples=True):
    """Yields per-example predictions of the best ensemble, one per input example (batches of at most the training
    batch size, a partial last batch included): logits (+ probabilities / class_ids for MultiClassHead, logistic for
    BinaryClassHead, predictions for RegressionHead)."""
    import torch
    self._restore_for_inference(input_fn)
    plan = self._ensemble_eval_plan()
    for item in input_utils.iterate_input_fn(input_fn):
      features = item[0] if isinstance(item, tuple) else item
      plan.run(input_utils.to_matrix(features, self._feature_keys), None)
      b = plan.rows
      logits = plan.ens_logits[:b]
      out = {"logits": logits.cpu().numpy()}
      if self._head.loss_kind == "softmax_xent":
        out["probabilities"] = torch.softmax(logits, dim=1).cpu().numpy()
        out["class_ids"] = logits.argmax(dim=1, keepdim=True).cpu().numpy()
      elif self._head.loss_kind == "sigmoid_xent":
        out["logistic"] = torch.sigmoid(logits).cpu().numpy()
      else:
        out["predictions"] = out["logits"]
      if predict_keys:
        out = {k: v for k, v in out.items() if k in predict_keys}
      if yield_single_examples:
        for i in range(b):
          yield {k: v[i] for k, v in out.items()}
      else:
        yield out

  def export_saved_model(self, *args, **kwargs):
    raise NotImplementedError("TF SavedModel export is outside the hot-path scope (SURVEY.md section 2); "
                              "the trained ensemble is in model_dir/ensemble-latest.npz + architecture-*.json")

  def get_variable_value(self, name):
    if name == "global_step":
      return self._global_step
    raise KeyError(name)
