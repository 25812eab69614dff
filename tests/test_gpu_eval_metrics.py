"""The streaming evaluation metrics on the GPU: adn_metrics_group against the independent NumPy restatement
(tests/metrics_oracle.py) and its own properties, the Evaluator ranking by auc / precision / recall / PR-AUC through the
Estimator, Estimator.evaluate's metric keys, and the same selection on two ranks.

Sum bounds: the kernel adds fp32 values widened to fp64 in an order fixed by (rows, dim, ops), the oracle in NumPy's
order; each order is within (n - 1) 2^-53 sum|v| of the exact sum, so the two differ by at most 2 n 2^-53 sum|v|.  A
binary head's predictions are the kernel's own fp32 logistic values (expf, <= 2 ulp), the oracle's NumPy fp32 ones
(<= 1 ulp): their sums may further differ by 8 2^-24 sum p.  Counts are exact: the synthetic logits are resampled so no
logistic value lies within 1e-6 of a threshold and no logit within 1e-6 of 0."""

import ctypes
import os
import socket

import numpy as np
import pytest

from tests import metrics_oracle as mo
from tests.test_gpu_inference import EB, _est_data, _input_fn, _make_estimator, fmt  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED, WORKSPACE = -22, -95, -12
NAMES = ("precision", "recall", "auc", "auc_precision_recall", "prediction/mean", "label/mean", "accuracy_baseline")


def _open():
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  return torch, _lib, lib


def clean_logits(rng, n, scale=3.0):
  """logits whose fp32 logistic is 1e-6 clear of every threshold and that are 1e-6 clear of 0"""
  x = (rng.standard_normal(n) * scale).astype(np.float32)
  thr = mo.thresholds().astype(np.float64)
  while True:
    p = mo.logistic32(x).astype(np.float64)
    bad = (np.abs(p[:, None] - thr[None, :]) < 1e-6).any(axis=1) | (np.abs(x) < 1e-6)
    if not bad.any():
      return x
    x[bad] = (rng.standard_normal(int(bad.sum())) * scale).astype(np.float32)


class Acc:
  """Device accumulators of n ops and the call that feeds them."""

  def __init__(self, torch, _lib, lib, n, binary):
    self.torch, self._lib, self.lib, self.binary = torch, _lib, lib, binary
    self.counts = torch.zeros((n, _lib.METRICS_COUNTS), dtype=torch.int64, device="cuda")
    self.sums = torch.zeros((n, 3), dtype=torch.float64, device="cuda")

  def ops(self, xs, ys, dims):
    _lib = self._lib
    kind = _lib.METRICS_BINARY if self.binary else _lib.METRICS_MEANS
    return (_lib.MetricsOp * len(xs))(*[
        _lib.MetricsOp(kind, 0, x.data_ptr(), y.data_ptr(), d, self.counts[i].data_ptr() if self.binary else None,
                       self.sums[i].data_ptr()) for i, (x, y, d) in enumerate(zip(xs, ys, dims))])

  def call(self, xs, ys, dims, rows, ws_bytes=None):
    _lib, torch = self._lib, self.torch
    need = _lib.query(_lib.Q_METRICS_WS, rows, max(dims), len(xs))
    ws = torch.empty((need,), dtype=torch.uint8, device="cuda")
    rc = self.lib.adn_metrics_group(self.ops(xs, ys, dims), len(xs), rows, ws.data_ptr(),
                                    need if ws_bytes is None else ws_bytes, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc

  def host(self):
    return self.counts.cpu().numpy(), self.sums.cpu().numpy()


def _dev(torch, a):
  return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def check_sums(got, x, y, pred, tag):
  n = x.size
  want = [np.sum(pred.astype(np.float64)), np.sum(y.astype(np.float64)), n]
  for k, (g, w, v) in enumerate(zip(got, want, (pred, y, np.ones(1)))):
    bound = 2 * n * 2.0 ** -53 * np.sum(np.abs(v.astype(np.float64)))
    if k == 0 and pred is not x:
      bound += 8 * 2.0 ** -24 * np.sum(np.abs(pred.astype(np.float64)))
    assert abs(g - w) <= bound, "%s sums[%d]: %r vs %r (bound %g)" % (tag, k, g, w, bound)


@pytest.mark.parametrize("rows", [1, 1000, 32768 + 17])
def test_binary_kernel_matches_oracle(rows):
  torch, _lib, lib = _open()
  rng = np.random.default_rng(rows)
  x = clean_logits(rng, rows)
  y = (rng.random(rows) < 0.35).astype(np.float32)
  acc = Acc(torch, _lib, lib, 1, True)
  assert acc.call([_dev(torch, x)], [_dev(torch, y)], [1], rows) == 0
  c, s = acc.host()
  want_c, _ = mo.counts_and_sums(x, y, True)
  np.testing.assert_array_equal(c[0], want_c)
  check_sums(s[0], x, y, mo.logistic32(x), "binary rows %d" % rows)


@pytest.mark.parametrize("dim", [1, 96])
def test_means_kernel_matches_oracle(dim):
  torch, _lib, lib = _open()
  rng = np.random.default_rng(dim)
  rows = 32768
  x = (rng.standard_normal((rows, dim)) * 2).astype(np.float32)
  y = rng.standard_normal((rows, dim)).astype(np.float32)
  acc = Acc(torch, _lib, lib, 1, False)
  assert acc.call([_dev(torch, x)], [_dev(torch, y)], [dim], rows) == 0
  _, s = acc.host()
  check_sums(s[0], x, y, x, "means dim %d" % dim)


def test_binary_kernel_nan_inf_and_huge_logits():
  """NaN: below every threshold and not a predicted positive; +inf and huge positive: p = 1, the top bucket 199;
  -inf and huge negative: p = 0, bucket 1 (0 > t_0 = -1e-7)."""
  torch, _lib, lib = _open()
  x = np.array([np.nan, np.inf, -np.inf, 1e30, -1e30, 88.0, -104.0, 0.0, np.nan, 3e38], dtype=np.float32)
  y = np.array([1, 1, 0, 1, 0, 0, 1, 1, 0, 1], dtype=np.float32)
  acc = Acc(torch, _lib, lib, 1, True)
  assert acc.call([_dev(torch, x)], [_dev(torch, y)], [1], x.size) == 0
  c, s = acc.host()
  np.testing.assert_array_equal(c[0], mo.counts_and_sums(x, y, True)[0])
  B = _lib.METRICS_THRESHOLDS + 1
  assert c[0][B + 0] == 1 and c[0][0] == 1          # the two NaNs, a positive and a negative
  assert c[0][B + 199] == 3 and c[0][1] == 2         # inf, 1e30, 3e38 / -inf, -1e30
  assert c[0][2 * B] == 1 and c[0][2 * B + 1] == 3   # 88 / inf, 1e30, 3e38
  assert np.isnan(s[0][0]) and s[0][1] == 6.0 and s[0][2] == 10.0


def test_many_ops_equal_single_ops_and_reruns_are_bit_identical():
  torch, _lib, lib = _open()
  rng = np.random.default_rng(11)
  rows, n = 5000, 40          # two launch groups of ops
  xs = [clean_logits(rng, rows) for _ in range(n)]
  ys = [(rng.random(rows) < 0.5).astype(np.float32) for _ in range(n)]
  dx, dy = [_dev(torch, v) for v in xs], [_dev(torch, v) for v in ys]
  group = Acc(torch, _lib, lib, n, True)
  assert group.call(dx, dy, [1] * n, rows) == 0
  gc, gs = group.host()
  for i in range(n):
    one = Acc(torch, _lib, lib, 1, True)
    assert one.call([dx[i]], [dy[i]], [1], rows) == 0
    oc, os_ = one.host()
    np.testing.assert_array_equal(gc[i], oc[0])
    assert gs[i].tobytes() == os_[0].tobytes()
  again = Acc(torch, _lib, lib, n, True)
  assert again.call(dx, dy, [1] * n, rows) == 0
  ac, as_ = again.host()
  assert ac.tobytes() == gc.tobytes() and as_.tobytes() == gs.tobytes()


@pytest.mark.parametrize("binary", [True, False])
def test_accumulation_over_batches_equals_one_call(binary):
  torch, _lib, lib = _open()
  rng = np.random.default_rng(5)
  dim = 1 if binary else 96
  sizes = [4096, 4096, 1000, 17]
  rows = sum(sizes)
  x = clean_logits(rng, rows) if binary else rng.standard_normal(rows * dim).astype(np.float32)
  x = x.reshape(rows, dim)
  y = (rng.random((rows, dim)) < 0.4).astype(np.float32)
  whole = Acc(torch, _lib, lib, 1, binary)
  assert whole.call([_dev(torch, x)], [_dev(torch, y)], [dim], rows) == 0
  parts = Acc(torch, _lib, lib, 1, binary)
  r0 = 0
  for b in sizes:
    assert parts.call([_dev(torch, x[r0:r0 + b])], [_dev(torch, y[r0:r0 + b])], [dim], b) == 0
    r0 += b
  wc, ws = whole.host()
  pc, ps = parts.host()
  np.testing.assert_array_equal(wc, pc)
  assert ps[0][2] == ws[0][2] == rows * dim
  pred = mo.logistic32(x) if binary else x
  for k, v in ((0, pred), (1, y)):
    assert abs(ps[0][k] - ws[0][k]) <= 4 * rows * dim * 2.0 ** -53 * np.sum(np.abs(v.astype(np.float64)))


def test_rejected_calls_change_no_accumulator():
  torch, _lib, lib = _open()
  rows = 64
  x, y = _dev(torch, np.zeros(rows * 2)), _dev(torch, np.zeros(rows * 2))
  acc = Acc(torch, _lib, lib, 2, True)
  acc.counts.fill_(7)
  acc.sums.fill_(3.5)
  before = _lib.launch_count()
  need = _lib.query(_lib.Q_METRICS_WS, rows, 1, 2)
  ws = torch.empty((need,), dtype=torch.uint8, device="cuda")
  sp = torch.cuda.current_stream().cuda_stream

  def call(ops, n=2, rows_=rows, ws_ptr=ws.data_ptr(), ws_bytes=need):
    return lib.adn_metrics_group(ops, n, rows_, ws_ptr, ws_bytes, sp)

  def good():
    return acc.ops([x, x], [y, y], [1, 1])

  cases = []
  ops = good(); ops[1].logits = None; cases.append((INVALID, call(ops)))
  ops = good(); ops[1].labels_f = None; cases.append((INVALID, call(ops)))
  ops = good(); ops[1].counts = None; cases.append((INVALID, call(ops)))
  ops = good(); ops[1].sums = None; cases.append((INVALID, call(ops)))
  ops = good(); ops[1].dim = 0; cases.append((INVALID, call(ops)))
  ops = good(); ops[1].dim = 2; cases.append((UNSUPPORTED, call(ops)))
  ops = good(); ops[1].kind = 5; cases.append((INVALID, call(ops)))
  ops = good(); ops[1].sums = ops[0].sums; cases.append((INVALID, call(ops)))
  cases.append((INVALID, call(good(), n=0)))
  cases.append((INVALID, call(good(), n=1025)))
  cases.append((INVALID, call(good(), rows_=0)))
  cases.append((INVALID, call(good(), ws_ptr=None)))
  cases.append((WORKSPACE, call(good(), ws_bytes=need - 1)))
  torch.cuda.synchronize()
  assert [w for w, _ in cases] == [g for _, g in cases]
  assert _lib.launch_count() == before
  assert (acc.counts == 7).all() and (acc.sums == 3.5).all()
  assert call(good()) == 0


# ------------------------------------------------------------------------------------------------------------------
# through the Estimator
# ------------------------------------------------------------------------------------------------------------------
def _spy(monkeypatch):
  """records, per plan and head, the GPU's own ensemble logits of every streamed hold-out batch and the trained state
  they were computed from (each candidate's mixture weights and members; the previous ensemble's)"""
  from adanet_b200.core import engine as eng
  seen = dict(cands=[], prev=[])
  step, prev_step = eng.IterationPlan.stream_eval_step, eng.EnsembleEvalPlan.stream_eval_step

  def params(nets):
    return [(n.numpy_params(), n.image_shape if n.stem else None, n.complexity) for n in nets]

  def cand(self, x, y):
    if not seen["cands"] or seen["cands"][-1]["plan"] is not self:
      seen["cands"].append(dict(plan=self, outs=[[] for _ in self.heads], state=self.state_dict(),
                                members=[params(h.member_nets) for _, h, _ in self.heads]))
    step(self, x, y)
    b = int(np.asarray(x).shape[0])
    for j, out in enumerate(self._metrics.ens_out):
      seen["cands"][-1]["outs"][j].append(out[:b].cpu().numpy())

  def prev(self, x, y):
    if not seen["prev"] or seen["prev"][-1]["plan"] is not self:
      seen["prev"].append(dict(plan=self, outs=[], members=params(self.members), w=self.mix_w.cpu().numpy(),
                               bias=self.bias.cpu().numpy(), gammas=list(self.gammas)))
    prev_step(self, x, y)
    seen["prev"][-1]["outs"].append(self.ens_logits[:self.rows].cpu().numpy())

  monkeypatch.setattr(eng.IterationPlan, "stream_eval_step", cand)
  monkeypatch.setattr(eng.EnsembleEvalPlan, "stream_eval_step", prev)
  return seen


def _logits64(members, w, bias, gammas, xh, yh, f16):
  """float64 ensemble logits of a trained VECTOR ensemble over the hold-out batches, with the bound of the GPU's
  logits around them (test_gpu_inference.wb_reference: the layer-by-layer error bound of the plane GEMMs)."""
  from tests.test_gpu_inference import F16_FLOOR, wb_reference
  ms = [dict(ws=p[0], bs=p[1], image=img) for p, img, _ in members]
  case = dict(C=1, head="sigmoid_xent", mix="vector")
  es, errs = [], []
  for i in range(0, xh.shape[0], EB):
    e, e_err, _, _ = wb_reference(case, ms, w, bias, xh[i:i + EB], yh[i:i + EB], gammas, F16_FLOOR if f16 else 0.0, False)
    es.append(np.reshape(e, -1))
    errs.append(np.reshape(e_err, -1))
  return np.concatenate(es), np.concatenate(errs)


def _from_buckets(bucket, cls_pos, pos):
  """the four ranked metrics from per-example buckets (number of thresholds below p) and predicted classes, by the
  oracle's formulas"""
  over = bucket[:, None] > np.arange(mo.NUM_THRESHOLDS)[None, :]
  tp, fp = (over & pos[:, None]).sum(0), (over & ~pos[:, None]).sum(0)
  tn, fn = (~pos).sum() - fp, pos.sum() - tp
  tpc, fpc = int((cls_pos & pos).sum()), int((cls_pos & ~pos).sum())
  return {"auc": mo.auc_roc(tp, fp, tn, fn), "auc_precision_recall": mo.auc_pr(tp, fp, fn),
          "precision": tpc / (tpc + fpc) if tpc + fpc else 0.0, "recall": tpc / pos.sum() if pos.sum() else 0.0}


def check_against_f64(metric, got, e, e_err, yh, tag, max_combos=4096):
  """The ranked value against float64 logits e (GPU logits within e +- e_err).  An example is ambiguous when its widened
  logistic interval [sigmoid(e - e_err), sigmoid(e + e_err)] +- 1e-6 (the fp32 logistic's own rounding) holds a
  threshold (for auc / auc_precision_recall), or its logit interval holds 0 (for precision / recall).  Bounds: each
  ambiguous example moves auc by at most 1/P (a positive) or 1/N (a negative) and recall by at most 1/P; k ambiguous
  class ids move precision by at most k / (PP - k), PP the predicted positives.  Where the ambiguous examples leave
  at most `max_combos` assignments, the value must also be one of those assignments' values exactly."""
  thr = mo.thresholds().astype(np.float64)
  sig = lambda v: 1.0 / (1.0 + np.exp(-v))
  nb = lambda p: (p[:, None] > thr[None, :]).sum(1)
  pos = np.reshape(yh, -1) > 0.5
  P, N = int(pos.sum()), int((~pos).sum())
  b_lo, b_hi, b_mid = nb(sig(e - e_err) - 1e-6), nb(sig(e + e_err) + 1e-6), nb(sig(e))
  c_lo, c_hi = e - e_err > 0, e + e_err > 0
  ref = _from_buckets(b_mid, e > 0, pos)[metric]
  if metric in ("auc", "auc_precision_recall"):
    amb = np.flatnonzero(b_lo != b_hi)
    options = [range(b_lo[i], b_hi[i] + 1) for i in amb]
  else:
    amb = np.flatnonzero(c_lo != c_hi)
    options = [(False, True)] * len(amb)
  bound = {"auc": (pos[amb].sum() / P if P else 0) + ((~pos)[amb].sum() / N if N else 0),
           "recall": pos[amb].sum() / P if P else 0,
           "precision": len(amb) / max(int((e > 0).sum()) - len(amb), 1) if len(amb) else 0.0}.get(metric)
  if bound is not None:
    assert abs(got - ref) <= bound + 1e-12, "%s %s: %r vs float64 %r, bound %g" % (tag, metric, got, ref, bound)
  n_combos = int(np.prod([len(o) for o in options])) if len(options) else 1
  if n_combos > max_combos:
    return
  vals = []
  for combo in np.array(np.meshgrid(*options, indexing="ij")).reshape(len(options), -1).T if len(options) else [()]:
    b, c = b_mid.copy(), e > 0
    if metric in ("auc", "auc_precision_recall"):
      b[amb] = combo
    else:
      c[amb] = np.asarray(combo, dtype=bool)
    vals.append(_from_buckets(b, c, pos)[metric])
  assert min(abs(got - v) for v in vals) <= 1e-12 * max(1.0, abs(got)), \
      "%s %s: %r is none of the %d float64 values %r" % (tag, metric, got, len(vals), sorted(set(vals))[:8])


def _close(got, want, tag):
  assert got == pytest.approx(want, rel=1e-12, abs=1e-14), "%s: %r vs oracle %r" % (tag, got, want)


@pytest.mark.parametrize("metric", ["auc", "precision", "recall", "auc_precision_recall"])
def test_evaluator_ranks_by_streaming_metric(fmt, metric, monkeypatch):
  """A BinaryClassHead Estimator with Evaluator(metric, maximize) over a hold-out input ending in a partial batch, two
  iterations: every ranked value (each candidate's, and the previous ensemble's at iteration 1) equals the oracle on
  the GPU's own ensemble logits, agrees with float64 logits of the trained state within check_against_f64's bounds,
  and the winner is their nanargmax."""
  import adanet_b200 as adanet
  from adanet_b200 import _lib
  from tests.test_gpu_inference import gamma32
  f16 = _lib.plane_format() == _lib.PLANES_F16
  seen = _spy(monkeypatch)
  x, y = _est_data("sigmoid", EB * 8, 1)
  xh, yh = _est_data("sigmoid", EB * 2 + 24, 3)
  ev = adanet.Evaluator(input_fn=_input_fn(xh, yh, "x"), metric_name=metric, objective="maximize")
  est = _make_estimator("sigmoid", None, evaluator=ev)
  est.train(_input_fn(x, y, "x"), max_steps=8)
  reps = est._search.reports
  assert len(reps) == 2 and len(seen["cands"]) == 2 and len(seen["prev"]) == 1
  for t, (rep, rec) in enumerate(zip(reps, seen["cands"])):
    vals = list(rep.ema_losses)
    cand_vals = vals[1:] if t else vals
    plan = rec["plan"]
    for j, (_, h, _) in enumerate(plan.heads):
      tag = "%s iteration %d %s" % (fmt, t, h.name)
      logits = np.concatenate(rec["outs"][j])
      assert logits.shape[0] == xh.shape[0]
      _close(cand_vals[j], mo.binary_metrics(logits, yh)[metric], tag)
      key = "c%d_" % next(c.index for c in plan.candidates if c.ehead is h)
      gam = [gamma32(0.01, 0.002, cx) for _, _, cx in rec["members"][j]]
      e, e_err = _logits64(rec["members"][j], rec["state"][key + "mix0"], rec["state"][key + "bias"], gam, xh, yh, f16)
      assert (np.abs(np.reshape(logits, -1) - e) <= e_err).all(), tag + ": ensemble logits outside the float64 bound"
      check_against_f64(metric, cand_vals[j], e, e_err, yh, tag)
    if t:
      pr = seen["prev"][0]
      _close(vals[0], mo.binary_metrics(np.concatenate(pr["outs"]), yh)[metric], "previous_ensemble")
      e, e_err = _logits64(pr["members"], pr["w"], pr["bias"], pr["gammas"], xh, yh, f16)
      check_against_f64(metric, vals[0], e, e_err, yh, "%s previous_ensemble" % fmt)
    assert rep.best_index == int(np.nanargmax(np.asarray(vals, dtype=np.float32)))


def test_auc_and_adanet_loss_pick_different_winners():
  """On this hold-out set ranking by auc keeps the linear candidate at iteration 0 where ranking by adanet_loss picks
  the one with a hidden layer: the Evaluator metric decides the search, as in the reference."""
  import adanet_b200 as adanet
  x, y = _est_data("sigmoid", EB * 8, 1)
  xh, yh = _est_data("sigmoid", EB * 2 + 24, 3)
  best = {}
  for metric, objective in (("auc", "maximize"), ("adanet_loss", "minimize")):
    ev = adanet.Evaluator(input_fn=_input_fn(xh, yh, "x"), metric_name=metric, objective=objective)
    est = _make_estimator("sigmoid", None, evaluator=ev)
    est.train(_input_fn(x, y, "x"), max_steps=8)
    best[metric] = est._search.reports[0].best_index
  assert best == {"auc": 0, "adanet_loss": 1}


def test_streaming_metric_routing_errors():
  """auc on a multi-class head and precision on a regression head raise ValueError when the Evaluator runs; an
  unknown name NotImplementedError."""
  import adanet_b200 as adanet
  for kind, metric, err in (("softmax", "auc", ValueError), ("mse", "precision", ValueError),
                            ("sigmoid", "roc", NotImplementedError)):
    x, y = _est_data(kind, EB * 4, 1)
    ev = adanet.Evaluator(input_fn=_input_fn(x, y, "x"), metric_name=metric, objective="maximize")
    est = _make_estimator(kind, None, evaluator=ev)
    with pytest.raises(err):
      est.train(_input_fn(x, y, "x"), max_steps=4)


def _eval_logits(est, xe):
  preds = list(est.predict(lambda: ({"x": xe[i:i + EB]} for i in range(0, xe.shape[0], EB))))
  return np.stack([p["logits"] for p in preds])


@pytest.mark.parametrize("kind", ["sigmoid", "mse", "mse96", "softmax"])
def test_evaluate_reports_head_metrics(fmt, kind, tmp_path):
  """evaluate() over 2.5 batches adds the v2 head's metrics, equal to the oracle on the ensemble's own logits;
  a MultiClassHead adds none."""
  import adanet_b200 as adanet
  from adanet_b200 import graph, train
  from adanet_b200.examples import simple_dnn
  if kind == "mse96":
    rng = np.random.default_rng(1)
    x = rng.standard_normal((EB * 8, 20)).astype(np.float32)
    y = (x @ rng.standard_normal((20, 96)).astype(np.float32) * 0.2).astype(np.float32)
    gen = simple_dnn.Generator(feature_columns=[graph.numeric_column("x", 20)],
                               optimizer=train.GradientDescentOptimizer(0.05), layer_size=16, seed=7)
    est = adanet.Estimator(head=adanet.heads.RegressionHead(label_dimension=96), subnetwork_generator=gen,
                           max_iteration_steps=4, model_dir=str(tmp_path))
    xe, ye = x[:EB * 2 + EB // 2], y[:EB * 2 + EB // 2]
  else:
    x, y = _est_data(kind, EB * 8, 1)
    xe, ye = _est_data(kind, EB * 2 + EB // 2, 2)
    est = _make_estimator(kind, str(tmp_path))
  est.train(_input_fn(x, y, "x"), max_steps=8)
  ev = est.evaluate(_input_fn(xe, ye, "x"))
  logits = _eval_logits(est, xe)
  if kind == "softmax":
    assert not set(NAMES) & set(ev)
    return
  want = mo.binary_metrics(logits, ye) if kind == "sigmoid" else mo.regression_metrics(logits, ye)
  assert set(want) <= set(ev)
  for k, v in want.items():
    if kind == "sigmoid" and k == "prediction/mean":
      # the mean of the kernel's expf logistic values against NumPy's: 8 2^-24 relative (module docstring)
      assert abs(ev[k] - v) <= 8 * 2.0 ** -24 * abs(v), "%s %s: %r vs oracle %r" % (kind, k, ev[k], v)
    else:
      _close(ev[k], v, "%s %s" % (kind, k))
  assert {"loss", "average_loss"} <= set(ev)


def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return s.getsockname()[1]


def _rank_worker(rank, world, port, model_dir, one, q):
  import torch
  import torch.distributed as dist
  os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
  os.environ["RANK"], os.environ["WORLD_SIZE"] = str(rank), str(world)
  if torch.cuda.device_count() >= world:
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  else:
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    q.put((rank, _auc_search(model_dir, one)))
  finally:
    dist.destroy_process_group()


def _one_candidate_estimator(model_dir, evaluator):
  """_make_estimator("sigmoid") whose generator offers only its first candidate: with balanced placement over two
  ranks, rank 1 owns no candidate ensemble"""
  import adanet_b200 as adanet
  from adanet_b200 import graph, train
  from adanet_b200.examples import simple_dnn
  from tests.test_gpu_inference import ED

  class OneCandidate(simple_dnn.Generator):
    def generate_candidates(self, *args, **kwargs):
      return super().generate_candidates(*args, **kwargs)[:1]

  gen = OneCandidate(feature_columns=[graph.numeric_column("x", ED)], optimizer=train.GradientDescentOptimizer(0.05),
                     layer_size=16, learn_mixture_weights=True, seed=7)
  ens = adanet.ensemble.ComplexityRegularizedEnsembler(optimizer=train.GradientDescentOptimizer(0.05), adanet_lambda=0.01,
                                                       adanet_beta=0.002, mixture_weight_type="vector", use_bias=True)
  return adanet.Estimator(head=adanet.heads.BinaryClassHead(), subnetwork_generator=gen, max_iteration_steps=4,
                          ensemblers=[ens], max_iterations=2, model_dir=model_dir, evaluator=evaluator)


def _auc_search(model_dir, one=False):
  import adanet_b200 as adanet
  x, y = _est_data("sigmoid", EB * 8, 1)
  xh, yh = _est_data("sigmoid", EB * 2 + 24, 3)
  ev = adanet.Evaluator(input_fn=_input_fn(xh, yh, "x"), metric_name="auc", objective="maximize")
  est = _one_candidate_estimator(model_dir, ev) if one else _make_estimator("sigmoid", model_dir, evaluator=ev)
  est.train(_input_fn(x, y, "x"), max_steps=8)
  return [(int(r.best_index), [float(v) for v in r.ema_losses]) for r in est._search.reports]


@pytest.mark.parametrize("one", [False, True], ids=["two_candidates", "one_candidate"])
def test_two_ranks_select_like_one(built_lib, tmp_path, one):
  """Balanced placement over two ranks (two GPUs, or both on cuda:0 over gloo): the same winners, and the same
  ranked auc values up to the fp32 all-gather of the candidate values.  With one candidate, rank 1 owns no candidate
  ensemble and streams its hold-out batches through no metric launch."""
  import torch.multiprocessing as mp
  single = _auc_search(str(tmp_path / "one"), one)
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, str(tmp_path / "two"), one, q)) for r in range(2)]
  for p in procs:
    p.start()
  got = dict(q.get(timeout=240) for _ in procs)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  for rank in (0, 1):
    assert [b for b, _ in got[rank]] == [b for b, _ in single]
    for (_, v2), (_, v1) in zip(got[rank], single):
      np.testing.assert_allclose(v2, np.float32(v1), rtol=0, atol=1e-6)
