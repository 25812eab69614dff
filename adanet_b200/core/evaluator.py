"""adanet.Evaluator mirror (adanet/core/evaluator.py:31-140): picks the best candidate
ensemble on a hold-out `input_fn` instead of the training-time EMA."""

import numpy as np


class Evaluator(object):
  """Evaluates candidate ensemble performance."""

  class Objective(object):
    MINIMIZE = "minimize"
    MAXIMIZE = "maximize"

  def __init__(self, input_fn, metric_name="adanet_loss", objective=Objective.MINIMIZE, steps=None):
    self._input_fn = input_fn
    self._steps = steps
    self._metric_name = metric_name
    self._objective = objective
    if objective == self.Objective.MINIMIZE:
      self._objective_fn = np.nanargmin
    elif objective == self.Objective.MAXIMIZE:
      self._objective_fn = np.nanargmax
    else:
      raise ValueError("Evaluator objective must be one of MINIMIZE or MAXIMIZE.")

  @property
  def input_fn(self):
    return self._input_fn

  @property
  def steps(self):
    return self._steps

  @property
  def metric_name(self):
    return self._metric_name

  @property
  def objective_fn(self):
    return self._objective_fn

  def evaluate(self, evaluate_batch_fn, num_candidates):
    """Streams up to `steps` batches of `input_fn` through `evaluate_batch_fn(features, labels)`
    (which returns one metric value per candidate for that batch) and returns the per-candidate
    mean, like the tf.metrics.mean accumulators of evaluator.py:97-140: "adanet_loss" and "loss" are
    per-batch scalars, weighted per batch (eval_metrics.py:120); "average_loss" and "accuracy" are
    weighted by the batch's example count, so a partial last batch counts for its examples."""
    from adanet_b200.core.input_utils import batch_size_of, iterate_input_fn
    per_example = self._metric_name in ("average_loss", "accuracy")
    sums = np.zeros((num_candidates,), dtype=np.float64)
    n, weight = 0, 0.0
    for features, labels in iterate_input_fn(self._input_fn):
      if self._steps is not None and n == self._steps:
        break
      w = float(batch_size_of(features)) if per_example else 1.0
      sums += w * np.asarray(evaluate_batch_fn(features, labels), dtype=np.float64)
      n += 1
      weight += w
    if n == 0:
      raise ValueError("Evaluator input_fn produced no batches")
    return list(sums / weight)

  def evaluate_streaming(self, add_batch_fn, values_fn):
    """The metrics that are not means of per-batch values (auc, precision, recall, ...: core/metrics.STREAM_METRICS):
    streams up to `steps` batches of `input_fn` through `add_batch_fn(features, labels)`, which adds each to the
    candidates' confusion counts and sums, then returns `values_fn()`, one finalized value per candidate (the
    streaming Keras metrics of evaluator.py:97-140)."""
    from adanet_b200.core.input_utils import iterate_input_fn
    n = 0
    for features, labels in iterate_input_fn(self._input_fn):
      if self._steps is not None and n == self._steps:
        break
      add_batch_fn(features, labels)
      n += 1
    if n == 0:
      raise ValueError("Evaluator input_fn produced no batches")
    return list(values_fn())
