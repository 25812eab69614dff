"""SimpleCNN search space: the `simple_cnn` subnetworks of BASELINE config 4.

Mirrors `SimpleCNNBuilder` / `SimpleCNNGenerator` of the reference's tutorial
(adanet/examples/tutorials/customizing_adanet.ipynb): one convolutional subnetwork per iteration (or one per seed,
for the 4-candidate configuration), every one the same architecture

  Conv2D(16, 3, padding="same", relu) -> MaxPool2D(2, 2) -> Flatten -> Dense(64, relu) -> Dense(logits)

with he_normal kernels, constant complexity 1, a Momentum(0.9) optimizer under cosine decay of the iteration step,
and mixture weights that are not trained (the deprecated `build_mixture_weights_train_op` returns a no-op).
The engine runs the conv/pool/flatten stem as one fused CUDA kernel (csrc/conv_stem.cu) and the dense layers on
the tensor-core plane pipeline.
"""

from __future__ import annotations

import functools

import adanet_b200 as adanet
from adanet_b200 import graph
from adanet_b200 import train


class SimpleCNNBuilder(adanet.subnetwork.Builder):
  """Builds a CNN subnetwork for AdaNet."""

  def __init__(self, learning_rate, max_iteration_steps, seed, name="simple_cnn"):
    self._learning_rate = learning_rate
    self._max_iteration_steps = max_iteration_steps
    self._seed = seed
    self._name = name

  def build_subnetwork(self, features, logits_dimension, training, iteration_step, summary, previous_ensemble=None):
    images = list(features.values())[0]
    summary.image("images", images)
    kernel_initializer = graph.he_normal_initializer(seed=self._seed)
    x = graph.layers.Conv2D(filters=16, kernel_size=3, padding="same", activation="relu",
                            kernel_initializer=kernel_initializer)(images)
    x = graph.layers.MaxPool2D(pool_size=2, strides=2)(x)
    x = graph.layers.Flatten()(x)
    x = graph.layers.Dense(units=64, activation="relu", kernel_initializer=kernel_initializer)(x)
    # the Head applies the softmax
    logits = graph.layers.Dense(units=logits_dimension, activation=None, kernel_initializer=kernel_initializer)(x)
    # constant complexity: all subnetworks share architecture and hyperparameters
    return adanet.Subnetwork(last_layer=x, logits=logits, complexity=1, persisted_tensors={})

  def build_subnetwork_train_op(self, subnetwork, loss, var_list, labels, iteration_step, summary, previous_ensemble=None):
    learning_rate = train.cosine_decay(learning_rate=self._learning_rate, global_step=iteration_step,
                                       decay_steps=self._max_iteration_steps)
    optimizer = train.MomentumOptimizer(learning_rate, .9)
    # NOTE: the Estimator increments the global step.
    return optimizer.minimize(loss=loss, var_list=var_list)

  def build_mixture_weights_train_op(self, loss, var_list, logits, labels, iteration_step, summary):
    return train.no_op("mixture_weights_train_op")

  @property
  def name(self):
    return self._name


class SimpleCNNGenerator(adanet.subnetwork.Generator):
  """Generates `num_candidates` SimpleCNNs at each iteration (1 = the tutorial's generator).

  The tutorial changes the seed with the iteration so that each subnetwork learns something different; with several
  candidates per iteration (BASELINE config 4) candidate j of iteration t gets seed + t * num_candidates + j and the
  name `simple_cnn_{j}` (names must be unique within an iteration, adanet/core/iteration.py:621-623)."""

  def __init__(self, learning_rate, max_iteration_steps, seed=None, num_candidates=1):
    if num_candidates < 1:
      raise ValueError("num_candidates must be >= 1")
    self._seed = seed
    self._num_candidates = int(num_candidates)
    self._builder_fn = functools.partial(SimpleCNNBuilder, learning_rate=learning_rate,
                                         max_iteration_steps=max_iteration_steps)

  def generate_candidates(self, previous_ensemble, iteration_number, previous_ensemble_reports, all_reports):
    n = self._num_candidates
    if n == 1:
      seed = self._seed
      if seed is not None:
        seed += iteration_number
      return [self._builder_fn(seed=seed)]
    return [self._builder_fn(seed=None if self._seed is None else self._seed + iteration_number * n + j,
                             name="simple_cnn_{}".format(j)) for j in range(n)]
