#!/usr/bin/env python
"""Throughput of the BASELINE.json configs that are not bench.py's headline line (configs[1], [3], [4]).

  python tools/bench_configs.py --config 4 [--batch B] [--steps K] [--warmup W] [--oracle-steps S]
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
      tools/bench_configs.py --config 4

Same metric and timing rules as bench.py (candidate-train examples/sec of one AdaNet iteration: every step trains
every candidate of the iteration; device time by CUDA events around K graph-replayed steps after W warm-up steps,
max over ranks; dataset resident in HBM and larger than L2), one JSON line per run on rank 0.  `--oracle-steps S`
also times S steps of the NumPy oracle on the host cores (rank 0) as the CPU reference for that config.

  config 2: adanet.Estimator-style search 784 -> H^L -> 10, (L, H) in {(1,64),(2,64),(1,128),(2,128)}, B=8192
  config 4: simple_cnn subnetworks (conv3x3x16+ReLU -> maxpool2 -> dense 64 -> 10) x 4 seeds, 32x32x3 synthetic,
            Momentum(0.9) + cosine decay, B=1024 (the tutorial's 64 is launch-latency bound; both are reported)
  config 5: 32-candidate sweep 100 -> H^L -> 10, L in 1..8 x H in {128,256,512,1024}, B=4096
"""

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def build_space(cfg, steps):
  from tests import parity_util as pu
  if cfg == 2:
    d, c = 784, 10
    cfgs = [(1, 64), (2, 64), (1, 128), (2, 128)]
    return d, c, (lambda t, which: pu.make_specs(cfgs, d, c, t, ("sgd", 0.05))[which]), "uniform"
  if cfg == 4:
    img = (32, 32, 3)
    opt = ("momentum_cosine", 0.003, 0.9, steps)
    return int(np.prod(img)), 10, (lambda t, which: pu.make_cnn_specs((0, 1, 2, 3), img, 16, 64, 10, t, opt)[which]), "images"
  if cfg == 5:
    d, c = 100, 10
    cfgs = [(L, H) for L in range(1, 9) for H in (128, 256, 512, 1024)]
    return d, c, (lambda t, which: pu.make_specs(cfgs, d, c, t, ("sgd", 0.01))[which]), "tabular"
  raise SystemExit("--config must be 2, 4 or 5")


def train_flops(specs):
  total = 0
  for s in specs:
    dims = list(s.dims)
    total += 6 * sum(a * b for a, b in zip(dims[:-1], dims[1:]))
    if getattr(s, "image_shape", None) is not None:
      h, w, cin = s.image_shape
      total += 4 * h * w * 9 * cin * np.shape(s.ws[0])[3]       # conv fwd + kernel gradient (no dX: first layer)
    else:
      total -= 2 * dims[0] * dims[1]                              # no dX for the input layer
  return int(total)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--config", type=int, required=True)
  ap.add_argument("--batch", type=int, default=0)
  ap.add_argument("--steps", type=int, default=100)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--rows", type=int, default=0)
  ap.add_argument("--oracle-steps", type=int, default=0)
  ap.add_argument("--placement", default="balanced", choices=["balanced", "round_robin", "sharded"])
  a = ap.parse_args()
  import torch
  import torch.distributed as dist
  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local = int(os.environ.get("LOCAL_RANK", "0"))
  torch.cuda.set_device(local)
  if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  from adanet_b200.distributed import exchange as ex
  from tests.parity_util import orc
  B = a.batch or {2: 8192, 4: 1024, 5: 4096}[a.config]
  in_dim, C, mk, kind = build_space(a.config, a.steps + a.warmup)
  # dataset larger than the 50 MB L2, resident in HBM
  rows = a.rows or max(8 * B, int(2.6e8 // (4 * in_dim)) // B * B)
  g = torch.Generator(device="cuda").manual_seed(1234)
  x = (torch.rand((rows, in_dim), device="cuda", generator=g) * 2 - 1) if kind != "tabular" else \
      torch.randn((rows, in_dim), device="cuda", generator=g)
  y = torch.randint(0, C, (rows,), device="cuda", generator=g)
  s = srch.AdaNetSearch(lambda t, frozen: mk(t, 1), eng.EnsemblerPlanSpec(optimizer=("sgd", 0.01), adanet_lambda=0.01),
                        in_dim, C, B, keep_traces=False, placement=a.placement)
  plan = s.build_iteration()
  batches = srch.consecutive_batches(x, y, B)
  for _ in range(a.warmup):
    plan.train_step(*next(batches))
  torch.cuda.synchronize()
  if world > 1:
    dist.barrier()
  l0 = _lib.launch_count()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(a.steps):
    plan.train_step(*next(batches))
  e1.record()
  torch.cuda.synchronize()
  if world > 1:
    dist.barrier()
  secs = ex.max_over_ranks(e0.elapsed_time(e1) * 1e-3, device=torch.device("cuda", local))
  launches = plan.launches_per_step
  # end of the iteration: all_gather of the candidates' EMA losses, selection, broadcast of the winner (SURVEY.md 8e)
  t0 = time.perf_counter()
  rep = s.finish_iteration()
  torch.cuda.synchronize()
  finish_ms = ex.max_over_ranks((time.perf_counter() - t0) * 1e3, device=torch.device("cuda", local))
  if rank == 0:
    specs = mk(0, 1)
    flops = train_flops(specs)
    out = {"metric": "candidate-train examples/sec per AdaNet iteration", "config": a.config, "candidates": len(specs),
           "batch": B, "n_gpus": world, "steps": a.steps, "warmup": a.warmup, "ms_per_step": secs / a.steps * 1e3,
           "value": B * a.steps / secs, "unit": "examples/s", "train_flops_per_example": flops,
           "useful_tflops": flops * B * a.steps / secs / 1e12, "launches_per_step_rank0": launches,
           "placement": a.placement, "finish_iteration_ms": finish_ms, "selected": rep.candidate_names[rep.best_index],
           "data": "synthetic, %d rows x %d resident in HBM (> L2)" % (rows, in_dim)}
    if a.oracle_steps:
      # the NumPy oracle on the host cores: same candidates, same batch size, bounded number of steps
      xs = x[:B * a.oracle_steps].cpu().numpy()
      ys = y[:B * a.oracle_steps].cpu().numpy()
      if kind == "images":
        xs = xs.reshape(-1, 32, 32, 3)
      cands = orc.build_candidates(0, mk(0, 0), [], orc.EnsemblerSpec(optimizer=("sgd", 0.01), adanet_lambda=0.01), C, 0.9)
      orc.train_step(cands, [], orc.EnsemblerSpec(optimizer=("sgd", 0.01), adanet_lambda=0.01), xs[:B], ys[:B])   # warm-up
      t0 = time.perf_counter()
      for i in range(a.oracle_steps):
        orc.train_step(cands, [], orc.EnsemblerSpec(optimizer=("sgd", 0.01), adanet_lambda=0.01), xs[i * B:(i + 1) * B],
                       ys[i * B:(i + 1) * B])
      dt = time.perf_counter() - t0
      out["cpu_baseline"] = {"value": B * a.oracle_steps / dt, "unit": "examples/s", "cores": os.cpu_count(), "kind": "port",
                             "sample": "%d steps of B=%d, NumPy oracle (BLAS threads = all cores)" % (a.oracle_steps, B)}
    print(json.dumps(out), flush=True)
  if world > 1:
    dist.destroy_process_group()


if __name__ == "__main__":
  main()
