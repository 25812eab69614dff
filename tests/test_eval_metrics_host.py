"""Host checks of the streaming evaluation metrics (core/metrics.py, Evaluator.evaluate_streaming): known answers
worked out by hand, the ROC trapezoid against the Mann-Whitney statistic, the package finalize against the
independent restatement in tests/metrics_oracle.py, metric-name routing and streaming over a ragged last batch."""

import numpy as np
import pytest

from adanet_b200.core import engine as eng
from adanet_b200.core import metrics as M
from adanet_b200.core.evaluator import Evaluator
from tests import metrics_oracle as mo

B = M.BUCKETS


def counts_of(neg, pos, cls_fp=0, cls_tp=0):
  """counts from {bucket: examples} of negatives and positives."""
  c = np.zeros((M.COUNTS,), dtype=np.int64)
  for b, k in neg.items():
    c[b] += k
  for b, k in pos.items():
    c[B + b] += k
  c[2 * B], c[2 * B + 1] = cls_fp, cls_tp
  return c


def test_perfect_separation_auc_is_one():
  r = M.finalize(counts_of({1: 5}, {199: 3}, cls_fp=0, cls_tp=3), [0.0, 3.0, 8.0])
  assert r["auc"] == 1.0 and r["precision"] == 1.0 and r["recall"] == 1.0
  # precision is 1 at every threshold below the positives' bucket, and recall runs from 1 to 0: the PR area is 1
  assert r["auc_precision_recall"] == pytest.approx(1.0, abs=1e-12)


@pytest.mark.parametrize("bucket", [1, 57, 199])
def test_one_bucket_auc_is_half(bucket):
  assert M.finalize(counts_of({bucket: 4}, {bucket: 6}), [0.0, 6.0, 10.0])["auc"] == 0.5


def test_div_no_nan_zeros():
  # no positives: recall and both areas are 0; no predicted positives: precision is 0
  r = M.finalize(counts_of({3: 4, 150: 2}, {}, cls_fp=0, cls_tp=0), [1.0, 0.0, 6.0])
  assert r["recall"] == 0.0 and r["precision"] == 0.0 and r["auc"] == 0.0 and r["auc_precision_recall"] == 0.0
  assert r["label/mean"] == 0.0 and r["accuracy_baseline"] == 1.0
  r = M.finalize(counts_of({}, {10: 3}), [1.0, 3.0, 3.0])
  assert r["precision"] == 0.0 and r["recall"] == 0.0 and r["auc"] == 0.0
  assert M.finalize(None, [0.0, 0.0, 0.0]) == {"prediction/mean": 0.0, "label/mean": 0.0}


def test_pr_auc_by_hand():
  """One negative in bucket 100, one positive in bucket 150 and one in bucket 50.  tp / fp / P = tp + fp per threshold:
     i < 50:        tp 2, fp 1, P 3;   50 <= i < 100: tp 1, fp 1, P 2;   100 <= i < 150: tp 1, fp 0, P 1;   i >= 150: 0.
  Only the steps at i = 49, 99 and 149 contribute (dtp = 0 elsewhere, or the slope is 0):
     i = 49:  dtp 1, dp 1, slope 1, intercept 1 - 2 = -1, ratio 3/2, denominator tp + fn = 2:  (1 - ln 1.5) / 2
     i = 99:  dtp 0 -> 0
     i = 149: dtp 1, dp 1, slope 1, intercept 0 - 0 = 0, P[150] = 0 so ratio 1, denominator 2:  1 / 2."""
  r = M.finalize(counts_of({100: 1}, {150: 1, 50: 1}), [0.0, 2.0, 3.0])
  assert r["auc_precision_recall"] == pytest.approx((1 - np.log(1.5)) / 2 + 0.5, abs=1e-15)
  # ROC: the negative sits between the two positives, so one of the two pairs is ordered: 1/2
  assert r["auc"] == 0.5


def mann_whitney(neg, pos):
  """P(bucket of a positive > bucket of a negative) + P(equal) / 2 from average ranks (NumPy only)."""
  scores = np.concatenate([neg, pos]).astype(np.float64)
  order = np.argsort(scores, kind="stable")
  ranks = np.empty_like(scores)
  ranks[order] = np.arange(1, scores.size + 1)
  for v in np.unique(scores):            # ties get their average rank
    m = scores == v
    ranks[m] = ranks[m].mean()
  n1, n0 = len(pos), len(neg)
  return (ranks[n0:].sum() - n1 * (n1 + 1) / 2) / (n1 * n0)


@pytest.mark.parametrize("seed", range(6))
def test_roc_trapezoid_is_mann_whitney(seed):
  """With every example in buckets 1..199 the ROC curve runs from (1, 1) to (0, 0) and each trapezoid counts the
  pairs of a negative bucket with half the same-bucket positives: the area is the Mann-Whitney statistic."""
  rng = np.random.default_rng(seed)
  neg = rng.integers(1, 200, size=rng.integers(1, 400))
  pos = rng.integers(1 + seed * 20, 200, size=rng.integers(1, 400))
  c = counts_of({}, {})
  np.add.at(c, neg, 1)
  np.add.at(c, B + pos, 1)
  assert abs(M.finalize(c, [0.0, 0.0, 1.0])["auc"] - mann_whitney(neg, pos)) <= 1e-12


def oracle_from_counts(c):
  """tp / fp / tn / fn by explicit loops over the buckets (an example in bucket b is above thresholds 0..b-1)."""
  tp, fp = np.zeros(200, np.int64), np.zeros(200, np.int64)
  for i in range(200):
    for b in range(i + 1, B):
      fp[i] += c[b]
      tp[i] += c[B + b]
  n, p = c[:B].sum(), c[B:2 * B].sum()
  return tp, fp, n - fp, p - tp


@pytest.mark.parametrize("seed", range(4))
def test_finalize_matches_oracle(seed):
  rng = np.random.default_rng(100 + seed)
  c = rng.integers(0, 50, size=M.COUNTS).astype(np.int64) * (rng.random(M.COUNTS) < 0.3)
  c[2 * B], c[2 * B + 1] = rng.integers(0, 20), rng.integers(0, 20)
  s = [rng.random() * 100, rng.random() * 50, 300.0]
  r = M.finalize(c, s)
  tp, fp, tn, fn = oracle_from_counts(c)
  assert r["auc"] == pytest.approx(mo.auc_roc(tp, fp, tn, fn), rel=1e-13, abs=1e-15)
  assert r["auc_precision_recall"] == pytest.approx(mo.auc_pr(tp, fp, fn), rel=1e-13, abs=1e-15)
  p = c[B:2 * B].sum()
  assert r["recall"] == (c[2 * B + 1] / p if p else 0.0)
  assert r["prediction/mean"] == s[0] / 300.0 and r["label/mean"] == s[1] / 300.0


def test_oracle_counts_agree_with_per_example_metrics():
  """The oracle's accumulator restatement, finalized by the package, equals its own per-example metric dict."""
  rng = np.random.default_rng(7)
  x = (rng.standard_normal(999) * 3).astype(np.float32)
  y = (rng.random(999) < 0.4).astype(np.float32)
  c, s = mo.counts_and_sums(x, y, True)
  got, want = M.finalize(c, s), mo.binary_metrics(x, y)
  for k in want:
    assert got[k] == pytest.approx(want[k], rel=1e-12, abs=1e-15), k


HEADS = ("softmax_xent", "mse", "sigmoid_xent")


@pytest.mark.parametrize("head", HEADS)
def test_metric_name_routing(head):
  """Each name a v2 head reports runs on that head; each name another head reports raises ValueError; an unknown name
  raises NotImplementedError.  The streaming names are kept apart from engine.EVAL_METRICS."""
  assert not set(M.STREAM_METRICS) & set(eng.EVAL_METRICS)
  reports = {"softmax_xent": {"adanet_loss", "loss", "average_loss", "accuracy"},
             "mse": {"adanet_loss", "loss", "average_loss", "prediction/mean", "label/mean"},
             "sigmoid_xent": {"adanet_loss", "loss", "average_loss", "accuracy", "precision", "recall", "auc",
                              "auc_precision_recall", "prediction/mean", "label/mean", "accuracy_baseline"}}[head]

  def route(metric):
    if metric in M.STREAM_METRICS:
      M.check_stream_metric(metric, head)
    else:
      eng._check_metric(metric, eng._HEAD_KIND[head])

  for metric in set(M.STREAM_METRICS) | set(eng.EVAL_METRICS):
    if metric in reports:
      route(metric)
    else:
      with pytest.raises(ValueError):
        route(metric)
  for metric in ("auc_roc", "f1", "precision/positive_threshold_0.5"):
    with pytest.raises(NotImplementedError):
      route(metric)


@pytest.mark.parametrize("binary", [True, False])
def test_streaming_ragged_last_batch(binary):
  """Evaluator.evaluate_streaming over batches of 64 ending in one of 13 equals one pass over all 333 examples, and
  `steps` stops it early."""
  rng = np.random.default_rng(3)
  x = (rng.standard_normal((333, 1)) * 2).astype(np.float32)
  y = (rng.random((333, 1)) < 0.3).astype(np.float32) if binary else rng.standard_normal((333, 1)).astype(np.float32)
  batches = [(x[i:i + 64], y[i:i + 64]) for i in range(0, 333, 64)]
  assert len(batches[-1][0]) == 13
  state = {"c": np.zeros(M.COUNTS, np.int64) if binary else None, "s": np.zeros(3)}

  def add(f, l):
    c, s = mo.counts_and_sums(f, l, binary)
    if binary:
      state["c"] += c
    state["s"] += s

  got = Evaluator(input_fn=lambda: batches).evaluate_streaming(add, lambda: [M.finalize(state["c"], state["s"])])[0]
  want = M.finalize(*mo.counts_and_sums(x, y, binary))
  assert got.keys() == want.keys()
  for k in want:
    assert got[k] == pytest.approx(want[k], rel=1e-14, abs=1e-16), k
  for k in ("auc", "auc_precision_recall", "precision", "recall"):
    if binary:
      assert got[k] == want[k]
  n = []
  Evaluator(input_fn=lambda: batches, steps=2).evaluate_streaming(lambda f, l: n.append(len(f)), lambda: [0.0])
  assert n == [64, 64]
  with pytest.raises(ValueError):
    Evaluator(input_fn=lambda: []).evaluate_streaming(add, lambda: [0.0])
