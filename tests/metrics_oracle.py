"""Independent NumPy restatement of the streaming binary / regression head metrics (test infrastructure only; the
package never imports it): per-example fp32 logistic values compared explicitly against each fp32 threshold of
tf.keras AUC(num_thresholds=200), and the Keras Precision / Recall / AUC / Mean formulas in fp64."""

import numpy as np

NUM_THRESHOLDS = 200


def thresholds() -> np.ndarray:
  """[0 - 1e-7, 1/199, ..., 198/199, 1 + 1e-7] as Keras builds them (Python floats), rounded to fp32."""
  t = [(i + 1) * 1.0 / (NUM_THRESHOLDS - 1) for i in range(NUM_THRESHOLDS - 2)]
  return np.asarray([0.0 - 1e-7] + t + [1.0 + 1e-7], dtype=np.float32)


def logistic32(logits) -> np.ndarray:
  x = np.asarray(logits, dtype=np.float32)
  with np.errstate(over="ignore"):
    return (np.float32(1.0) / (np.float32(1.0) + np.exp(-x))).astype(np.float32)


def _dnn(a, b):
  a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
  out = np.zeros(np.broadcast(a, b).shape)
  nz = b != 0
  np.divide(np.broadcast_to(a, out.shape), np.broadcast_to(b, out.shape), out=out, where=nz)
  return out


def confusion_from_p(p, labels):
  """(tp, fp, tn, fn) [200] int64 of fp32 scores p against labels (positive when > 0.5), by explicit comparison."""
  p = np.asarray(p, dtype=np.float32).reshape(-1)
  pos = np.asarray(labels, dtype=np.float32).reshape(-1) > 0.5
  with np.errstate(invalid="ignore"):
    above = p[:, None] > thresholds()[None, :]          # NaN compares False: predicted negative everywhere
  tp = (above & pos[:, None]).sum(axis=0).astype(np.int64)
  fp = (above & ~pos[:, None]).sum(axis=0).astype(np.int64)
  return tp, fp, (~pos).sum() - fp, pos.sum() - tp


def auc_roc(tp, fp, tn, fn) -> float:
  tpr = _dnn(tp, tp + fn)
  fpr = _dnn(fp, fp + tn)
  total = 0.0
  for i in range(NUM_THRESHOLDS - 1):
    total += (fpr[i] - fpr[i + 1]) * (tpr[i] + tpr[i + 1]) / 2.0
  return float(total)


def auc_pr(tp, fp, fn) -> float:
  """Keras interpolate_pr_auc, term by term."""
  total = 0.0
  for i in range(NUM_THRESHOLDS - 1):
    dtp = float(tp[i] - tp[i + 1])
    p0, p1 = float(tp[i] + fp[i]), float(tp[i + 1] + fp[i + 1])
    dp = max(p0 - p1, 0.0)
    slope = dtp / dp if dp != 0 else 0.0
    intercept = float(tp[i + 1]) - slope * p1
    ratio = p0 / p1 if (p0 > 0 and p1 > 0) else 1.0
    denom = max(float(tp[i + 1] + fn[i + 1]), 0.0)
    total += slope * (dtp + intercept * np.log(ratio)) / denom if denom != 0 else 0.0
  return float(total)


def binary_metrics(logits, labels) -> dict:
  """The metric dict of a BinaryClassHead's ensemble logits [n] or [n, 1] and labels."""
  x = np.asarray(logits, dtype=np.float32).reshape(-1)
  y = np.asarray(labels, dtype=np.float32).reshape(-1)
  p = logistic32(x)
  tp, fp, tn, fn = confusion_from_p(p, y)
  pos = y > 0.5
  with np.errstate(invalid="ignore"):
    pred_pos = x > 0
  tp_c, fp_c = int((pred_pos & pos).sum()), int((pred_pos & ~pos).sum())
  label_mean = float(np.sum(y.astype(np.float64)) / y.size)
  return {
      "precision": float(_dnn(tp_c, tp_c + fp_c)), "recall": float(_dnn(tp_c, pos.sum())),
      "auc": auc_roc(tp, fp, tn, fn), "auc_precision_recall": auc_pr(tp, fp, fn),
      "prediction/mean": float(np.sum(p.astype(np.float64)) / p.size), "label/mean": label_mean,
      "accuracy_baseline": max(label_mean, 1.0 - label_mean),
  }


def regression_metrics(logits, labels) -> dict:
  x = np.asarray(logits, dtype=np.float32).astype(np.float64)
  y = np.asarray(labels, dtype=np.float32).astype(np.float64)
  return {"prediction/mean": float(x.sum() / x.size), "label/mean": float(y.sum() / y.size)}


def counts_and_sums(logits, labels, binary: bool):
  """The accumulator state adn_metrics_group defines (include/adanet_b200.h) for one batch, restated: the 201-bucket
  histograms of negatives and positives (bucket = number of thresholds below p), the class-id counts and the sums."""
  x = np.asarray(logits, dtype=np.float32).reshape(-1)
  y = np.asarray(labels, dtype=np.float32).reshape(-1)
  if not binary:
    return None, np.array([x.astype(np.float64).sum(), y.astype(np.float64).sum(), x.size])
  p = logistic32(x)
  with np.errstate(invalid="ignore"):
    bucket = (p[:, None] > thresholds()[None, :]).sum(axis=1)
    pred_pos = x > 0
  pos = y > 0.5
  counts = np.zeros((2 * (NUM_THRESHOLDS + 1) + 2,), dtype=np.int64)
  np.add.at(counts, bucket[~pos], 1)
  np.add.at(counts, NUM_THRESHOLDS + 1 + bucket[pos], 1)
  counts[-2] = int((pred_pos & ~pos).sum())
  counts[-1] = int((pred_pos & pos).sum())
  return counts, np.array([p.astype(np.float64).sum(), y.astype(np.float64).sum(), x.size])
