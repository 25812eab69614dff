"""The AdaNet outer loop over the GPU iteration plan.

Arithmetic/bookkeeping skeleton of `Estimator.train`
(adanet/core/estimator.py:809-999) without the TF graph rebuilds: per
iteration build the candidates' plans on the GPUs that own them, run
`max_iteration_steps` steps, exchange the EMA losses, pick the best ensemble
(adanet/core/estimator.py:1415-1517), freeze its new subnetwork and continue.
`adanet_b200.Estimator` drives this class; `bench.py` and the parity tests use
it directly.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from adanet_b200.core import engine as eng
from adanet_b200.distributed import exchange as ex


def select_best_index(losses: Sequence[float], iteration: int, force_grow: bool = False,
                      replay_index: Optional[int] = None) -> int:
  """Estimator._get_best_ensemble_index without an Evaluator
  (adanet/core/estimator.py:1415-1517): replay override, single candidate -> 0,
  force_grow with two candidates -> 1, else np.nanargmin over the EMA adanet
  losses, dropping index 0 (the previous ensemble) under force_grow."""
  if replay_index is not None:
    return int(replay_index)
  if len(losses) == 1:
    return 0
  if iteration > 0 and force_grow and len(losses) == 2:
    return 1
  arr = np.asarray(losses, dtype=np.float32)
  if force_grow and iteration > 0:
    return int(np.nanargmin(arr[1:])) + 1
  return int(np.nanargmin(arr))


def in_graph_best_index(losses: Sequence[float]) -> int:
  """_IterationBuilder._best_candidate_index (adanet/core/iteration.py:1011-1046):
  argmin with NaN mapped to -inf (a NaN candidate wins, surfacing the NaN)."""
  arr = np.asarray(losses, dtype=np.float32).copy()
  if arr.size == 1:
    return 0
  arr[np.isnan(arr)] = -np.inf
  return int(np.argmin(arr))


@dataclass
class IterationReport:
  iteration: int
  candidate_names: List[str]          # [previous_ensemble?] + new candidates, reference order (iteration.py:603,725)
  ema_losses: List[float]
  best_index: int
  architecture: List[Tuple[int, str]]  # winner's (iteration, builder name) list (architecture.py)
  replay_indices: List[int]
  mixture_weights: np.ndarray
  bias: np.ndarray
  steps: int
  train_seconds: float                # device time of the train phase (CUDA events)
  traces: Optional[Dict[str, Dict[str, np.ndarray]]] = None


@dataclass
class EnsembleCandidate:
  """One candidate ensemble of an iteration (adanet/ensemble/strategy.py:26-76 `Candidate`): the strategy's
  candidate name, the new subnetworks it contains (indices into the iteration's builders) and whether the
  previous ensemble's subnetworks are kept."""
  name: str
  builders: List[int]
  # True: the whole previous ensemble, False: none of it, or the indices of the previous members to keep (partial
  # pruning by a custom Strategy, adanet/core/ensemble_builder.py:367-388)
  keep_previous: object = True
  ens_index: int = 0          # which of the search's ensemblers builds it (adanet/core/iteration.py:683-693)


def strategy_candidates(strategies: Sequence[str], builder_names: Sequence[str]) -> List[EnsembleCandidate]:
  """Grow / Solo / All (adanet/ensemble/strategy.py:79-117), in the order the strategies are listed."""
  out: List[EnsembleCandidate] = []
  for st in strategies:
    if st == "grow":
      out += [EnsembleCandidate("{}_grow".format(n), [i], True) for i, n in enumerate(builder_names)]
    elif st == "solo":
      out += [EnsembleCandidate("{}_solo".format(n), [i], False) for i, n in enumerate(builder_names)]
    elif st == "all":
      out.append(EnsembleCandidate("all", list(range(len(builder_names))), True))
    else:
      raise ValueError("unknown ensemble strategy %r" % (st,))
  return out


class AdaNetSearch:
  """Runs AdaNet iterations on this process's GPU (rank r of G owns candidates i % G == r)."""

  def __init__(self, search_space: Callable[[int, List[eng.DenseNet]], List[eng.SubnetworkPlanSpec]],
               ensembler: eng.EnsemblerPlanSpec, in_dim: int, logits_dim: int, batch_size: int,
               head: str = "softmax_xent", adanet_loss_decay: float = 0.9, force_grow: bool = False,
               replay_indices: Optional[Sequence[int]] = None, device: Optional[torch.device] = None,
               use_cuda_graph: bool = True, multi_stream: bool = True, keep_traces: bool = True,
               trace_capacity: int = 4096, placement: str = "balanced", strategies: Sequence[str] = ("grow",),
               candidates_fn: Optional[Callable] = None):
    # one EnsemblerPlanSpec or a list: every strategy candidate is built once per ensembler (iteration.py:683-693)
    self.search_space = search_space
    self.ensemblers = list(ensembler) if isinstance(ensembler, (list, tuple)) else [ensembler]
    if len({e.name for e in self.ensemblers}) != len(self.ensemblers):
      raise ValueError("ensemblers must have distinct names")
    self.winner_ens_index = 0          # ensembler of the current best ensemble
    self.in_dim, self.C, self.batch, self.head = in_dim, logits_dim, batch_size, head
    self.decay, self.force_grow = adanet_loss_decay, force_grow
    self.replay_indices = list(replay_indices) if replay_indices is not None else None
    self.device = device or torch.device("cuda", torch.cuda.current_device())
    self.use_cuda_graph, self.multi_stream = use_cuda_graph, multi_stream
    self.keep_traces, self.trace_capacity = keep_traces, trace_capacity
    if placement not in ("balanced", "round_robin", "sharded"):
      raise ValueError("placement must be 'balanced', 'round_robin' or 'sharded'")
    self.placement = placement
    # candidate ensembles of an iteration: candidates_fn(specs, n_frozen) -> [EnsembleCandidate], or the named strategies
    self.strategies = tuple(strategies)
    self.candidates_fn = candidates_fn
    self.frozen: List[eng.DenseNet] = []
    self.iteration = 0
    self.prev_best_ema: Optional[float] = None
    self.architecture: List[Tuple[int, str]] = []
    self.replay_trace: List[int] = []
    self.mixture_weights: Optional[np.ndarray] = None
    self.bias: Optional[np.ndarray] = None
    self.reports: List[IterationReport] = []
    self.plan: Optional[eng.IterationPlan] = None

  @property
  def ens(self) -> eng.EnsemblerPlanSpec:
    """The first (for single-ensembler searches: the only) ensembler."""
    return self.ensemblers[0]

  @ens.setter
  def ens(self, value: eng.EnsemblerPlanSpec):
    if len(self.ensemblers) != 1:
      raise NotImplementedError("replacing the ensembler of a multi-ensembler search")
    self.ensemblers = [value]

  @property
  def winner_ens(self) -> eng.EnsemblerPlanSpec:
    """The ensembler that built the current best ensemble (its mixture weights are `self.mixture_weights`)."""
    return self.ensemblers[self.winner_ens_index]

  # -- iteration assembly ------------------------------------------------------
  def build_iteration(self) -> eng.IterationPlan:
    specs = self.search_space(self.iteration, self.frozen)
    names = [s.name for s in specs]
    if len(set(names)) != len(names):
      dup = [n for n in names if names.count(n) > 1][0]
      raise ValueError("Two subnetworks have the same name '{}'".format(dup))   # iteration.py:621-623
    if not specs:
      raise ValueError("Each iteration must have at least one Builder.")      # iteration.py:564-565
    self._specs = specs
    g, r = ex.world(), ex.rank()
    # candidate ensembles (strategy candidates x this ensembler)
    ecs = (self.candidates_fn(specs, len(self.frozen)) if self.candidates_fn is not None
           else strategy_candidates(self.strategies, names))
    if not ecs:
      raise ValueError("the ensemble strategies produced no candidate")
    if len(self.ensemblers) > 1:      # strategy candidates x ensemblers, strategy-candidate major (iteration.py:683-693)
      ecs = [EnsembleCandidate(c.name, list(c.builders), c.keep_previous, j) for c in ecs for j in range(len(self.ensemblers))]
    self._check_kept_members(specs, ecs)
    self._ecands = ecs
    # subnetwork -> rank.  Subnetworks read by the same candidate ensemble (e.g. AllStrategy) must share a GPU --
    # splitting them would need the member logits gathered every step (SURVEY.md 8e) -- so the units of placement
    # are the connected components of "shares an ensemble"; a component's cost is its training FLOPs per example
    # (sum d_i d_{i+1}).  "balanced" = longest-processing-time first, "round_robin" = the reference-like i % G.
    costs = [sum(a * b for a, b in zip(s.dims[:-1], s.dims[1:])) +
             (s.image_shape[0] * s.image_shape[1] * int(np.prod(np.shape(s.ws[0])[:3])) * np.shape(s.ws[0])[3]
              if s.image_shape is not None else 0) for s in specs]
    default_grow = (len(self.ensemblers) == 1 and len(ecs) == len(specs) and all(
        c.keep_previous is True and c.builders == [i] and c.name == "{}_grow".format(specs[i].name) for i, c in enumerate(ecs)))
    shards = {}
    shardable = (self.placement == "sharded" and g > 1 and default_grow and self.ens.mixture_weight_type != "matrix"
                 and not any(getattr(s, "own_input", False) for s in specs))
    if shardable:
      # row-sharded placement (distributed/exchange.sharded_placement): a candidate heavier than a rank's fair share is
      # trained data-parallel by several ranks; its first rank reports it at the end of the iteration
      ranks = ex.sharded_placement(costs, g, self.batch)
      self._owners = [rk[0] for rk in ranks]
      mine = [i for i, rk in enumerate(ranks) if r in rk]
      for i, rk in enumerate(ranks):        # every rank creates every group, in the same order (new_group is collective)
        if len(rk) > 1:
          grp = ex.subgroup(rk)
          if r in rk:
            shards[i] = eng.ShardComm(rk, r, grp)
      self._shard_ranks = ranks
    else:
      self._owners = ex.component_owners(costs, [c.builders for c in ecs], g,
                                         "balanced" if self.placement == "sharded" else self.placement)
      mine = ex.owned_indices(len(specs), r, g, self._owners)
      self._shard_ranks = [[o] for o in self._owners]
    self._ec_owners = [self._owners[c.builders[0]] for c in ecs]
    local = None if default_grow else [(j, c.name, list(c.builders), c.keep_previous, self.ensemblers[c.ens_index])
                                       for j, c in enumerate(ecs) if self._ec_owners[j] == r]
    prev_ens_name = self.winner_ens.name if (self.frozen and len(self.ensemblers) > 1) else None
    self.plan = eng.IterationPlan(self.iteration, [specs[i] for i in mine], self.frozen, self.ens, self.batch,
                                  self.in_dim, self.C, self.head, self.decay, self.trace_capacity, self.device,
                                  candidate_indices=mine, use_cuda_graph=self.use_cuda_graph,
                                  multi_stream=self.multi_stream, prev_mixture_weights=self.mixture_weights,
                                  prev_bias=self.bias, ensemble_candidates=local, prev_ens_name=prev_ens_name,
                                  shards=shards)
    return self.plan

  def _check_kept_members(self, specs, ecs):
    """A candidate ensemble must keep every previous member that its new subnetworks, or the members it keeps, read:
    the winner's members are replayed from that list alone."""
    for c in ecs:
      kept = [self.frozen[i] for i in eng.kept_indices(c.keep_previous, len(self.frozen))]
      keys = {(f.iteration, f.name) for f in kept}
      reads = [(specs[b].name, key) for b in c.builders for key in eng.member_refs(getattr(specs[b], "inputs", None))]
      reads += [(f.name, key) for f in kept for key in eng.member_refs(f.inputs)]
      for who, key in reads:
        if tuple(key) not in keys:
          raise NotImplementedError("candidate ensemble %s drops %s (iteration %d) from the previous ensemble, but %s reads "
                                    "its hidden layers" % (c.name, key[1], key[0], who))

  def train_iteration(self, batches: Iterator, steps: int, on_step=None) -> float:
    """Runs `steps` training steps; returns device seconds (CUDA events) of the phase.

    The transfer of batch i+1 is started (copy stream) right after step i is enqueued, so host batches stream
    in under the kernels; `on_step(plan)` -- e.g. reading the step's losses back -- runs after that."""
    plan = self.plan or self.build_iteration()
    start = torch.cuda.Event(enable_timing=True)
    end = torch.cuda.Event(enable_timing=True)
    start.record()
    if steps > 0:
      plan.stage_batch(*next(batches))
    for i in range(steps):
      plan.train_step()
      if i + 1 < steps:
        plan.stage_batch(*next(batches))
      if on_step is not None:
        on_step(plan)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / 1e3

  def restart_on_tf32_if_overflowed(self) -> bool:
    """fp16 planes hold |v| < 65520 only (csrc/plane_fmt.cuh).  When any rank met a finite value beyond that during
    the iteration just trained, its results are discarded: the process switches to TF32 planes for good, the plan is
    dropped and the caller trains the iteration again (its candidates are re-created from the same deterministic
    specs).  Returns True in that case.  One all_reduce of a flag per iteration, outside the step."""
    from adanet_b200 import _lib
    plan = self.plan
    if plan is None or plan.fmt != _lib.PLANES_F16 or plan.xp is None:      # TF32 planes / fp32 SIMT path: nothing to fall back from
      return False
    # the input split, the optimizer and the head raise the sticky flag; a GEMM result beyond the range becomes Inf in
    # the planes and shows up as a non-finite loss, which is treated the same way (a candidate that truly diverged
    # costs one re-run of the iteration, after which the process stays on TF32 planes)
    local = plan.plane_overflow() or not all(np.isfinite(v) for v in plan.ema_losses())
    flag = ex.max_over_ranks(1.0 if local else 0.0, device=self.device) > 0.0
    if not flag:
      return False
    import logging
    logging.getLogger("adanet_b200").warning(
        "iteration %d: a value did not fit the fp16 split planes; re-running the iteration on TF32 planes", self.iteration)
    _lib.set_plane_format(_lib.PLANES_TF32)
    self.plan = None
    self.tf32_fallbacks = getattr(self, "tf32_fallbacks", 0) + 1
    return True

  def finish_iteration(self, train_seconds: float = 0.0, local_metric_fn=None, previous_metric=None,
                       objective_fn=None) -> IterationReport:
    """Selection + growth (bookkeeping phase, estimator.py:1247-1283).

    Without an Evaluator the candidates are compared on their EMA adanet losses
    (estimator.py:1491-1495).  With one, `local_metric_fn(plan)` returns the
    hold-out metric of each local candidate, `previous_metric` that of the
    previous ensemble, and `objective_fn` is np.nanargmin / np.nanargmax
    (estimator.py:1487-1490)."""
    plan, specs, t = self.plan, self._specs, self.iteration
    ecs, ec_owners = self._ecands, self._ec_owners
    k = len(ecs)
    g = ex.world()
    local = plan.ema_losses() if local_metric_fn is None else list(local_metric_fn(plan))
    new_losses = ex.gather_candidate_losses(local, k, device=self.device, owners=ec_owners)
    names = ["t{}_{}_{}".format(t, c.name, self.ensemblers[c.ens_index].name) for c in ecs]
    losses = list(new_losses)
    if t > 0:
      names = ["previous_ensemble"] + names
      losses = [self.prev_best_ema if local_metric_fn is None else previous_metric] + losses
    replay = None
    if self.replay_indices is not None and t < len(self.replay_indices):
      replay = self.replay_indices[t]
    if objective_fn is None or replay is not None or len(losses) == 1 or (t > 0 and self.force_grow and len(losses) == 2):
      best = select_best_index(losses, t, self.force_grow, replay)
    elif self.force_grow and t > 0:
      best = int(objective_fn(np.asarray(losses[1:], dtype=np.float32))) + 1
    else:
      best = int(objective_fn(np.asarray(losses, dtype=np.float32)))
    ema_all = (ex.gather_candidate_losses(plan.ema_losses(), k, device=self.device, owners=ec_owners)
               if local_metric_fn is not None else new_losses)
    traces = plan.traces() if self.keep_traces else None
    self.last_winner_index = None
    self.last_winner_builders, self.last_winner_keeps_previous = None, True
    self.last_winner_kept = None
    if t > 0 and best == 0:
      pass   # previous ensemble kept; nothing grows
    else:
      ci = best - (1 if t > 0 else 0)
      ec = ecs[ci]
      owner = ec_owners[ci]
      w_ens = self.ensemblers[ec.ens_index]
      matrix = w_ens.mixture_weight_type == "matrix"
      kept_idx = eng.kept_indices(ec.keep_previous, len(self.frozen))
      kept = [self.frozen[i] for i in kept_idx]
      # materialise the winner's new subnetworks on every rank for frozen replay
      if ex.rank() == owner:
        head = next(h for gidx, h, _ in plan.heads if gidx == ci)
        new_members = [next(c for c in plan.candidates if c.index == b).net for b in ec.builders]
        for k, m in enumerate(new_members):
          if m.batch != self.batch:      # trained on a row slice: frozen replay needs full-minibatch buffers
            ws_, bs_ = m.numpy_params()
            new_members[k] = eng.DenseNet(m.name, m.dims, ws_, bs_, m.complexity, self.batch, self.device, t, m.shared,
                                          m.image_shape, inputs=m.inputs, members=kept)
        mix_ws, bias = head.mixture_weight_tensors(), head.bias
      else:
        new_members = [eng.DenseNet(specs[b].name, specs[b].dims, specs[b].ws, specs[b].bs, specs[b].complexity,
                                    self.batch, self.device, t, specs[b].shared, specs[b].image_shape,
                                    inputs=getattr(specs[b], "inputs", None), members=kept)
                       for b in ec.builders]
        n_members = len(kept) + len(new_members)
        if matrix:
          mix_ws = [torch.empty((m.last_layer_dim, self.C), dtype=torch.float32, device=self.device)
                    for m in kept + new_members]
        else:
          wshape = (n_members,) if w_ens.mixture_weight_type == "scalar" else (n_members, self.C)
          mix_ws = [torch.empty(wshape, dtype=torch.float32, device=self.device)]
        bias = torch.empty((self.C,), dtype=torch.float32, device=self.device)
      ex.broadcast_tensors([t_ for m in new_members for t_ in m.all_params()] + mix_ws + [bias], src=owner)
      if ex.rank() != owner:
        for m in new_members:
          m.refresh_planes()   # their planes were split from the (pre-broadcast) initial weights
      self.frozen = kept + new_members
      self.architecture = [self.architecture[i] for i in kept_idx] + [(t, specs[b].name) for b in ec.builders]
      self.prev_best_ema = ema_all[ci]
      self.last_winner_index = ec.builders[-1]
      self.last_winner_builders, self.last_winner_keeps_previous = list(ec.builders), ec.keep_previous is not False
      self.last_winner_kept = list(kept_idx)
      self.last_winner_name = ec.name
      self.winner_ens_index = ec.ens_index
      # SCALAR [N] / VECTOR [N,C] array, or the list of N [D_k,C] matrices (MATRIX)
      self.mixture_weights = ([w.cpu().numpy().copy() for w in mix_ws] if matrix else mix_ws[0].cpu().numpy().copy())
      self.bias = bias.cpu().numpy().copy()
    self.replay_trace = self.replay_trace + [best]
    rep = IterationReport(t, names, [float(v) for v in losses], best, list(self.architecture),
                          list(self.replay_trace), self.mixture_weights, self.bias, plan.steps_done,
                          train_seconds, traces)
    self.reports.append(rep)
    self.iteration += 1
    self.plan = None
    return rep

  def run(self, batches: Iterator, steps_per_iteration: int, iterations: int) -> List[IterationReport]:
    for _ in range(iterations):
      while True:
        self.build_iteration()
        secs = self.train_iteration(batches, steps_per_iteration)
        if not self.restart_on_tf32_if_overflowed():
          break
      self.finish_iteration(secs)
    return self.reports


def consecutive_batches(x_all, y_all, batch_size: int) -> Iterator:
  """Consecutive slices in fixed order, wrapping at the end (SURVEY.md section 8d)."""
  n = x_all.shape[0]
  cursor = 0
  while True:
    if cursor + batch_size > n:
      cursor = 0
    yield x_all[cursor:cursor + batch_size], y_all[cursor:cursor + batch_size]
    cursor += batch_size
