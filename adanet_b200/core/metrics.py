"""Host finalize of the streaming evaluation metrics of the v2 BinaryClassHead and RegressionHead (adn_metrics_group,
include/adanet_b200.h): turns an ensemble's accumulated (counts, sums) into the metric values, in fp64, after the
tf.keras definitions those heads use (AUC(num_thresholds=200) with interpolation for the ROC and PR curves, Precision,
Recall, Mean).  Keras keeps its accumulators in float32; here the counts are exact int64 and the sums fp64."""

from typing import Dict, Optional

import numpy as np

THRESHOLDS = 200
BUCKETS = THRESHOLDS + 1
COUNTS = 2 * BUCKETS + 2      # negative histogram, positive histogram, (negatives, positives) with logit > 0

# the metrics the streaming path computes, and the heads (loss kinds) that report each of them
STREAM_METRICS = {
    "precision": ("sigmoid_xent",),
    "recall": ("sigmoid_xent",),
    "auc": ("sigmoid_xent",),
    "auc_precision_recall": ("sigmoid_xent",),
    "accuracy_baseline": ("sigmoid_xent",),
    "prediction/mean": ("sigmoid_xent", "mse"),
    "label/mean": ("sigmoid_xent", "mse"),
}


def check_stream_metric(metric: str, head: str):
  """Refuses a STREAM_METRICS metric that a head of loss kind `head` does not report."""
  if head not in STREAM_METRICS[metric]:
    raise ValueError("%s is not an evaluation metric of a %s head" % (metric, head))


def div_no_nan(a, b):
  a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
  return np.where(b == 0, 0.0, a / np.where(b == 0, 1.0, b))


def confusion(counts):
  """(tp, fp, tn, fn) at each of the THRESHOLDS thresholds, from the two bucket histograms: an example in bucket b is
  above thresholds 0..b-1, so tp_i / fp_i are the positives / negatives of the buckets past i."""
  counts = np.asarray(counts, dtype=np.int64)
  neg, pos = counts[:BUCKETS], counts[BUCKETS:2 * BUCKETS]
  tp = np.cumsum(pos[::-1])[::-1][1:]
  fp = np.cumsum(neg[::-1])[::-1][1:]
  return tp, fp, neg.sum() - fp, pos.sum() - tp


def roc_auc(tp, fp, tn, fn) -> float:
  """Keras AUC(curve="ROC", summation_method="interpolation"): trapezoids between consecutive thresholds."""
  recall = div_no_nan(tp, tp + fn)
  fpr = div_no_nan(fp, fp + tn)
  return float(np.sum((fpr[:-1] - fpr[1:]) * (recall[:-1] + recall[1:]) / 2.0))


def pr_auc(tp, fp, fn) -> float:
  """Keras AUC(curve="PR", summation_method="interpolation"): interpolate_pr_auc (Davis & Goadrich, 2006)."""
  tp, fp, fn = (np.asarray(v, dtype=np.float64) for v in (tp, fp, fn))
  dtp = tp[:-1] - tp[1:]
  p = tp + fp
  dp = p[:-1] - p[1:]
  slope = div_no_nan(dtp, np.maximum(dp, 0.0))
  intercept = tp[1:] - slope * p[1:]
  both = (p[:-1] > 0) & (p[1:] > 0)
  ratio = np.where(both, div_no_nan(p[:-1], np.maximum(p[1:], 0.0)), 1.0)
  return float(np.sum(div_no_nan(slope * (dtp + intercept * np.log(ratio)),
                                 np.maximum(tp[1:] + fn[1:], 0.0))))


def finalize(counts: Optional[np.ndarray], sums) -> Dict[str, float]:
  """The metric dict of one ensemble: with `counts` (a binary head) precision, recall, auc, auc_precision_recall,
  prediction/mean (of the logistic), label/mean and accuracy_baseline; without (a regression head) prediction/mean
  (of the logits over every element) and label/mean."""
  s = np.asarray(sums, dtype=np.float64)
  label_mean = float(div_no_nan(s[1], s[2]))
  out = {"prediction/mean": float(div_no_nan(s[0], s[2])), "label/mean": label_mean}
  if counts is None:
    return out
  counts = np.asarray(counts, dtype=np.int64)
  tp, fp, tn, fn = confusion(counts)
  fp_cls, tp_cls = counts[2 * BUCKETS], counts[2 * BUCKETS + 1]
  out.update({
      "precision": float(div_no_nan(tp_cls, tp_cls + fp_cls)),
      "recall": float(div_no_nan(tp_cls, counts[BUCKETS:2 * BUCKETS].sum())),
      "auc": roc_auc(tp, fp, tn, fn),
      "auc_precision_recall": pr_auc(tp, fp, fn),
      "accuracy_baseline": max(label_mean, 1.0 - label_mean),
  })
  return out
