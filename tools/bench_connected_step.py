"""Times an AdaNet iteration-1 training step whose 8 candidates read the frozen winner's last hidden layer at their
logits layer, alternated with the same plan without those pieces.

Workload: bench.py's configs[2] candidates (100->H->H->10, H in bench.WIDTHS) at B = 32768.  Iteration 0 trains the
plain candidates for a few steps and freezes the winner; iteration 1 is then built twice from candidate_weights(1):
  plain      the candidates as bench.py runs them
  connected  each candidate's logits layer reads concat([its own last hidden layer, the winner's last hidden layer]):
             the kernel gains the winner's width in rows (glorot-uniform, seeded), the forward is a multi-source plane
             GEMM and the backward adds one dW-only op per candidate to the logits-layer wave
Both plans are warmed up (the first step runs eagerly, the second captures the CUDA graph), then timed alternately in
rounds of --steps steps with CUDA events.  Prints the card name and power limit, the median step time of each plan
over the rounds and the launches per step, as one JSON line.

  python tools/bench_connected_step.py [--steps 100] [--rounds 5]
"""

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown"
  except Exception:
    return "unknown"


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=100)
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--iter0-steps", type=int, default=20)
  args = ap.parse_args()
  import torch
  import __graft_entry__ as g
  g.build()
  import bench
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  from oracle.adanet_oracle import make_tabular

  dev = torch.device("cuda", 0)
  x_np, y_np = make_tabular(bench.BATCH * 8, bench.IN_DIM, bench.CLASSES, seed=1234)
  x, y = torch.as_tensor(x_np).to(dev), torch.as_tensor(y_np).to(dev)
  ens = eng.EnsemblerPlanSpec(optimizer=("sgd", bench.ENS_LR), adanet_lambda=bench.LAMBDA, adanet_beta=bench.BETA)
  plain = lambda t, frozen: [eng.SubnetworkPlanSpec(n, d, cx, ("sgd", bench.SUB_LR), ws, bs)
                             for n, d, cx, ws, bs in bench.candidate_weights(t)]
  s = srch.AdaNetSearch(plain, ens, bench.IN_DIM, bench.CLASSES, bench.BATCH, device=dev, keep_traces=False)
  s.run(srch.consecutive_batches(x, y, bench.BATCH), args.iter0_steps, 1)
  win = s.frozen[-1]
  hw = win.dims[-2]

  def connected(t, frozen):
    out = []
    for k, spec in enumerate(plain(t, frozen)):
      h = spec.dims[-2]
      rng = np.random.default_rng(5000 + k)
      lim = np.sqrt(6.0 / (h + hw + bench.CLASSES))
      extra = rng.uniform(-lim, lim, size=(hw, bench.CLASSES)).astype(np.float32)
      spec.ws[-1] = np.concatenate([spec.ws[-1], extra], axis=0)
      spec.inputs = [None] * (len(spec.dims) - 2) + [[
          {"src": "own", "rows": [0, h]},
          {"src": "member", "iteration": win.iteration, "name": win.name, "layer": len(win.dims) - 3, "rows": [h, h + hw]}]]
      out.append(spec)
    return out

  plans = {}
  for name, space in (("plain", plain), ("connected", connected)):
    s.search_space = space
    plans[name] = s.build_iteration()
    s.plan = None
  batches = srch.consecutive_batches(x, y, bench.BATCH)
  for p in plans.values():
    for _ in range(3):
      p.train_step(*next(batches))
  torch.cuda.synchronize()
  times = {k: [] for k in plans}
  for _ in range(args.rounds):
    for name, p in plans.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(args.steps):
        p.train_step(*next(batches))
      e1.record()
      torch.cuda.synchronize()
      times[name].append(e0.elapsed_time(e1) / args.steps)
  for p in plans.values():
    assert np.isfinite(p.last_losses()).all(), "non-finite loss"
  print(json.dumps({
      "card": card(), "plane_format": "fp16" if _lib.plane_format() == _lib.PLANES_F16 else "tf32",
      "batch": bench.BATCH, "widths": list(bench.WIDTHS), "frozen_winner": [win.name, hw],
      "step_ms": {k: float(np.median(v)) for k, v in times.items()},
      "step_ms_rounds": {k: [round(t, 4) for t in v] for k, v in times.items()},
      "launches_per_step": {k: int(p.launches_per_step) for k, p in plans.items()}}), flush=True)


if __name__ == "__main__":
  main()
