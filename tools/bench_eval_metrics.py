"""Streaming evaluation metric measurements (adn_metrics_group), one JSON line per result:

  1. the kernel alone at rows = 32768, n in {1, 8, 32} ops: BINARY (dim 1) and MEANS (dim 1 and 96): us per call (CUDA
     events over many calls after warm-up) and launches per call.  It reads a few hundred KB per op and is bound by
     launch latency, not bandwidth, so no share of HBM bandwidth is reported;
  2. a hold-out pass of the bench's 8 candidates (100 -> h -> h -> 1, h = 64..1024) on a binary head, 16 batches of
     32768: ranked by adanet_loss (IterationPlan.eval_step, the per-batch mean) and by auc (the streaming path),
     alternated over 5 rounds; ms per pass (host clock around work that ends in a device synchronise), medians.

The card's name and power limit are read in the same run and printed first."""

import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROWS = 32768


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except Exception as e:   # noqa: BLE001
    out = "nvidia-smi unavailable: %s" % e
  return out


def kernel_bench(torch, lib, _lib, n, kind, dim, reps=200, warm=10):
  dev = torch.device("cuda")
  xs = [torch.randn((ROWS, dim), device=dev) * 3 for _ in range(n)]
  ys = [(torch.rand((ROWS, dim), device=dev) < 0.4).float() for _ in range(n)]
  counts = torch.zeros((n, _lib.METRICS_COUNTS), dtype=torch.int64, device=dev)
  sums = torch.zeros((n, 3), dtype=torch.float64, device=dev)
  wsb = _lib.query(_lib.Q_METRICS_WS, ROWS, dim, n)
  ws = torch.empty((wsb,), dtype=torch.uint8, device=dev)
  ops = (_lib.MetricsOp * n)(*[
      _lib.MetricsOp(kind, 0, x.data_ptr(), y.data_ptr(), dim,
                     counts[i].data_ptr() if kind == _lib.METRICS_BINARY else None, sums[i].data_ptr())
      for i, (x, y) in enumerate(zip(xs, ys))])
  sp = torch.cuda.current_stream().cuda_stream
  call = lambda: _lib.check(lib.adn_metrics_group(ops, n, ROWS, ws.data_ptr(), wsb, sp), "adn_metrics_group")
  for _ in range(warm):
    call()
  before = _lib.launch_count()
  call()
  launches = _lib.launch_count() - before
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record()
  for _ in range(reps):
    call()
  e1.record()
  torch.cuda.synchronize()
  return dict(kind="kernel", metrics="binary" if kind == _lib.METRICS_BINARY else "means", rows=ROWS, dim=dim, n=n,
              us=round(e0.elapsed_time(e1) * 1e3 / reps, 2), launches_per_call=launches)


def holdout_bench(torch, rounds=5, batches=16):
  import adanet_b200 as adanet
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  widths, D = (64, 128, 192, 256, 384, 512, 768, 1024), 100

  def space(t, frozen):
    out = []
    for i, h in enumerate(widths):
      dims = [D, h, h, 1]
      rng = np.random.default_rng(1000 + 100 * t + i)
      ws = [rng.uniform(-np.sqrt(6.0 / (a + b)), np.sqrt(6.0 / (a + b)), size=(a, b)).astype(np.float32)
            for a, b in zip(dims[:-1], dims[1:])]
      bs = [np.zeros((b,), np.float32) for b in dims[1:]]
      out.append(eng.SubnetworkPlanSpec("2_layer_dnn_w%d" % h, dims, float(np.sqrt(2.0)), ("sgd", 0.05), ws, bs,
                                        shared={"num_layers": 2}))
    return out

  dev = torch.device("cuda")
  rng = np.random.default_rng(1234)
  xh = torch.as_tensor(rng.standard_normal((ROWS * batches, D), dtype=np.float32)).to(dev)
  yh = torch.as_tensor((rng.random((ROWS * batches, 1)) < 0.4).astype(np.float32)).to(dev)
  holdout = [(xh[i * ROWS:(i + 1) * ROWS], yh[i * ROWS:(i + 1) * ROWS]) for i in range(batches)]
  ens = eng.EnsemblerPlanSpec(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001)
  s = srch.AdaNetSearch(space, ens, D, 1, ROWS, head="sigmoid_xent", device=dev, keep_traces=False)
  plan = s.build_iteration()
  for _ in range(3):
    plan.train_step(*holdout[0])
  ev_loss = adanet.Evaluator(input_fn=lambda: holdout, metric_name="adanet_loss")
  ev_auc = adanet.Evaluator(input_fn=lambda: holdout, metric_name="auc", objective="maximize")

  def by_loss():
    return ev_loss.evaluate(lambda f, l: plan.eval_step(f, l, "adanet_loss"), len(plan.heads))

  def by_auc():
    acc = plan.stream_metrics("auc")
    return ev_auc.evaluate_streaming(lambda f, l: plan.stream_eval_step(f, l), lambda: acc.values("auc"))

  def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    vals = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, vals

  timed(by_loss)
  timed(by_auc)
  tl, ta = [], []
  for _ in range(rounds):
    t, vl = timed(by_loss)
    tl.append(t)
    before = eng._lib.launch_count()
    t, va = timed(by_auc)
    auc_launches = eng._lib.launch_count() - before
    ta.append(t)
  return dict(kind="holdout_pass", candidates=len(plan.heads), batches=batches, rows=ROWS,
              adanet_loss_ms=[round(t, 2) for t in tl], auc_ms=[round(t, 2) for t in ta],
              adanet_loss_median_ms=round(float(np.median(tl)), 2), auc_median_ms=round(float(np.median(ta)), 2),
              auc_launches_per_pass=auc_launches, winner_by_loss=int(np.nanargmin(vl)), winner_by_auc=int(np.nanargmax(va)))


def main():
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  print(json.dumps({"card": card(), "plane_format": _lib.plane_format()}), flush=True)
  for n in (1, 8, 32):
    for kind, dim in ((_lib.METRICS_BINARY, 1), (_lib.METRICS_MEANS, 1), (_lib.METRICS_MEANS, 96)):
      print(json.dumps(kernel_bench(torch, lib, _lib, n, kind, dim)), flush=True)
  print(json.dumps(holdout_bench(torch)), flush=True)


if __name__ == "__main__":
  main()
