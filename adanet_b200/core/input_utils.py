"""input_fn conventions.

The reference's `input_fn` returns TF tensors / a tf.data.Dataset.  Here an
`input_fn()` returns an iterable (list, generator, DataLoader ...) of
`(features, labels)` minibatches, where `features` is an array [B, D] or a dict
of column key -> array [B, d_k] (NumPy or torch, host or device) and `labels`
an array [B] / [B, 1] (class ids) or [B, C] (regression / binary targets).
Training batches must all have the same size (a static-shape engine: ragged
tails are dropped with a warning, cf. `drop_remainder`).  Evaluation and
prediction take batches of up to that size, so a partial last batch counts.
"""

import logging

import numpy as np


def iterate_input_fn(input_fn):
  data = input_fn()
  if isinstance(data, tuple) and len(data) == 2 and not isinstance(data[0], tuple):
    # a single (features, labels) pair: one batch
    yield data
    return
  for item in data:
    yield item


def batch_size_of(features) -> int:
  if isinstance(features, dict):
    return int(next(iter(features.values())).shape[0])
  return int(features.shape[0])


def feature_widths(features):
  """Values per example of each feature ([B, d] -> d; NHWC images [B, H, W, C] -> H*W*C)."""
  if isinstance(features, dict):
    return {k: (int(np.prod(v.shape[1:])) if len(v.shape) > 1 else 1) for k, v in features.items()}
  return {"x": int(np.prod(features.shape[1:])) if len(features.shape) > 1 else 1}


def feature_shapes(features):
  """Per-example shape of each feature, kept for image features so builders see [batch, H, W, C] tensors."""
  if not isinstance(features, dict):
    features = {"x": features}
  return {k: tuple(int(d) for d in v.shape[1:]) or (1,) for k, v in features.items()}


def to_matrix(features, keys):
  """Concatenates the feature dict in `keys` order into one [B, D] array (input_layer)."""
  import torch
  if not isinstance(features, dict):
    return features
  parts = [features[k] for k in keys]
  parts = [p.reshape(p.shape[0], -1) for p in parts]
  if len(parts) == 1:
    return parts[0]
  if any(isinstance(p, torch.Tensor) for p in parts):
    return torch.cat([torch.as_tensor(p) for p in parts], dim=1)
  return np.concatenate([np.asarray(p) for p in parts], axis=1)


def warn_ragged(got, want):
  logging.warning("adanet_b200: dropping a ragged batch of %d examples (static batch size %d)", got, want)
