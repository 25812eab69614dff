"""Per-launch device-time profile of the benchmarked training step (bench.py, one GPU).

  python tools/step_profile.py --out DIR [--warmup 5] [--steps 3]

Builds the step's plan the way bench.py does (its data, weights and constants are imported from bench), warms it up
through its CUDA graph, times the graphed step with CUDA events, then profiles `--steps` eager steps
(plan.use_cuda_graph = False: every kernel of the step is attributed to its own launch) with torch.profiler.

For every launch position of the step it reports the kernel, its device time (median over the profiled steps) and
the wave it belongs to.  Plane GEMM launches also get the useful FLOPs and the algorithmic HBM bytes of their wave,
computed from the shapes below, and the bound with the fraction of it reached:
  * FLOP bound: the plane GEMM issues 3 fp16 MMAs per product (hi*hi, hi*lo', lo'*hi), so its floor is
    3 * useful FLOPs over the cuBLAS fp16 rate measured in the same run (bench.measure_cublas_peaks);
  * HBM bound: algorithmic bytes over bench.load_peaks()'s HBM bandwidth.  Operands and outputs are counted once,
    at their plane size (2 x 2 B per value in fp16, K padded to the 64-column k-block, plus the sign-bit words);
    dense fp32 outputs at 4 B per value.  Split-K partials and their reduction are not algorithmic and are not counted.
The fraction is floor / measured time.  Writes DIR/step_profile.json and prints a table.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

BK16 = 64                       # fp16 plane k-block (columns)


def _pad(n, m):
  return (n + m - 1) // m * m


def plane_bytes(rows, cols):
  """hi + lo' fp16 planes (cols padded to the k-block) + sign-bit words of a [rows, cols] tensor."""
  return rows * _pad(cols, BK16) * 4 + rows * _pad(cols, 32) // 8


def gemm_waves(batch=bench.BATCH, widths=bench.WIDTHS, d_in=bench.IN_DIM, classes=bench.CLASSES):
  """(wave label, EPI kind, useful FLOPs, algorithmic bytes) of every plane GEMM launch of one step, in launch order.
  Layer l of candidate H maps dims[l] -> dims[l + 1], dims = [d_in, H, H, classes]."""
  cands = [[d_in, h, h, classes] for h in widths]
  out = []
  for l in range(3):
    fl = sum(2 * batch * d[l] * d[l + 1] for d in cands)
    if l < 2:      # planes out (+ sign bits), bias
      by = sum(plane_bytes(batch, d[l]) + plane_bytes(d[l], d[l + 1]) + plane_bytes(batch, d[l + 1]) for d in cands)
    else:          # logits: dense fp32 out
      by = sum(plane_bytes(batch, d[l]) + plane_bytes(d[l], d[l + 1]) + batch * d[l + 1] * 4 for d in cands)
    out.append(("fwd L%d" % (l + 1), 0, fl, by))
  for k in range(3):
    l = 2 - k      # backward visits the logits layer first
    fl = sum(2 * batch * d[l] * d[l + 1] for d in cands)
    by = sum(plane_bytes(batch, d[l]) + plane_bytes(batch, d[l + 1]) + d[l] * d[l + 1] * 4 for d in cands)
    out.append(("bwd k=%d dW" % k, 2, fl, by))
    if l > 0:      # dX (planes out, ReLU mask of the layer input, column sums); the first layer has none
      by = sum(plane_bytes(batch, d[l + 1]) + plane_bytes(d[l], d[l + 1]) + batch * _pad(d[l], 32) // 8 +
               plane_bytes(batch, d[l]) + (batch + 31) // 32 * d[l] * 4 for d in cands)
      out.append(("bwd k=%d dX" % k, 1, fl, by))
  return out


def classify(name):
  m = re.search(r"pl_gemm_kernel<(\d+), (\d+)>", name)
  if m:
    return "gemm", int(m.group(2))
  for key, kind in (("reduce_partials", "reduce"), ("colsum", "colsum"), ("opt_step", "optimizer"),
                    ("step_increment", "optimizer"), ("split_kernel", "split"), ("head_bookkeeping", "bookkeeping"),
                    ("counter_add", "counter")):
    if key in name:
      return kind, None
  if "head" in name or "loss" in name:
    return "head", None
  return "other", None


def label_step(names):
  """Wave label of each launch of one step, from the launch order of Plan._enqueue_waves."""
  labels, fwd, bwd = [], 0, -1
  for n in names:
    kind, epi = classify(n)
    if kind == "gemm" and epi == 0:
      fwd += 1
      labels.append("fwd L%d" % fwd)
    elif kind == "gemm" and epi == 2:
      bwd += 1
      labels.append("bwd k=%d dW" % bwd)
    elif kind == "gemm":
      labels.append("bwd k=%d dX" % bwd)
    elif kind in ("reduce", "colsum"):
      labels.append("bwd k=%d %s" % (bwd, kind))
    elif kind == "split" and fwd == 0:
      labels.append("split x")
    else:
      labels.append(kind)
  return labels


def gpu_info():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except Exception as exc:
    return "nvidia-smi unavailable: %r" % (exc,)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", required=True)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--steps", type=int, default=3)
  ap.add_argument("--timed-steps", type=int, default=50)
  args = ap.parse_args()
  import torch
  from torch.profiler import ProfilerActivity, profile

  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  if _lib.plane_format() != _lib.PLANES_F16:
    raise SystemExit("step_profile: the FLOP and byte model is written for the fp16 plane format")
  dev = torch.device("cuda", 0)
  info = gpu_info()
  peaks = bench.measure_cublas_peaks(torch)
  hbm_gbs, _, _, hbm_src = bench.load_peaks()

  x_np, y_np = bench.make_tabular(bench.DATA_ROWS, bench.IN_DIM, bench.CLASSES, seed=1234)
  x_dev, y_dev = torch.as_tensor(x_np).to(dev), torch.as_tensor(y_np).to(dev)
  ens = eng.EnsemblerPlanSpec(optimizer=("sgd", bench.ENS_LR), adanet_lambda=bench.LAMBDA, adanet_beta=bench.BETA)
  space = lambda t, frozen: [eng.SubnetworkPlanSpec(n, d, cx, ("sgd", bench.SUB_LR), ws, bs, shared={"num_layers": 2})
                             for n, d, cx, ws, bs in bench.candidate_weights(t)]
  s = srch.AdaNetSearch(space, ens, bench.IN_DIM, bench.CLASSES, bench.BATCH, device=dev, keep_traces=False,
                        placement="balanced")
  plan = s.build_iteration()
  batches = srch.consecutive_batches(x_dev, y_dev, bench.BATCH)
  for _ in range(args.warmup):
    plan.train_step(*next(batches))
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(args.timed_steps):
    plan.train_step(*next(batches))
  e1.record()
  torch.cuda.synchronize()
  graph_ms = e0.elapsed_time(e1) / args.timed_steps

  plan.use_cuda_graph = False
  for _ in range(2):
    plan.train_step(*next(batches))
  torch.cuda.synchronize()
  per_step = plan.launches_per_step
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.steps):
      plan.train_step(*next(batches))
    torch.cuda.synchronize()
  kern = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "Memcpy" not in e.name
                 and "Memset" not in e.name), key=lambda e: e.time_range.start)
  if len(kern) != per_step * args.steps:
    raise SystemExit("step_profile: %d kernels for %d steps of %d launches" % (len(kern), args.steps, per_step))
  names = [e.name for e in kern[:per_step]]
  dur = np.array([[e.time_range.end - e.time_range.start for e in kern[i * per_step:(i + 1) * per_step]]
                  for i in range(args.steps)], dtype=np.float64)      # us
  for i in range(1, args.steps):
    if [e.name for e in kern[i * per_step:(i + 1) * per_step]] != names:
      raise SystemExit("step_profile: the launch sequence differs between steps")
  med = np.median(dur, axis=0)
  labels = label_step(names)
  model = {w[0]: w for w in gemm_waves()}
  f16 = peaks.get("f16_tflops")
  rows = []
  for i, (n, lab, us) in enumerate(zip(names, labels, med)):
    r = {"pos": i, "wave": lab, "kernel": n, "us": float(us)}
    if lab in model and classify(n)[0] == "gemm":
      _, _, fl, by = model[lab]
      t_flop = 3.0 * fl / (f16 * 1e12) if f16 else None
      t_hbm = by / (hbm_gbs * 1e9)
      bound = "FLOP" if (t_flop or 0.0) >= t_hbm else "HBM"
      floor = max(t_flop or 0.0, t_hbm)
      r.update({"useful_flops": fl, "bytes": by, "useful_tflops": fl / (us * 1e-6) / 1e12,
                "gbs": by / (us * 1e-6) / 1e9, "floor_us": floor * 1e6, "bound": bound,
                "frac_of_bound": floor / (us * 1e-6)})
    rows.append(r)
  total = float(med.sum())
  res = {"gpu": info, "cublas_peaks": peaks, "hbm_gbs": hbm_gbs, "hbm_source": hbm_src,
         "graph_step_ms": graph_ms, "eager_kernel_sum_ms": total / 1e3, "profiled_steps": args.steps,
         "launches_per_step": per_step, "launches": rows}
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "step_profile.json"), "w") as f:
    json.dump(res, f, indent=1)
  print("GPU: %s | cuBLAS fp16 %.0f TFLOP/s | HBM %.0f GB/s (%s)" % (info, f16 or float("nan"), hbm_gbs, hbm_src))
  print("graphed step %.3f ms; kernel time per eager step %.3f ms" % (graph_ms, total / 1e3))
  print("%3s %-16s %-44s %9s %6s %9s %5s %6s" % ("#", "wave", "kernel", "us", "%", "floor us", "bound", "frac"))
  for r in rows:
    kn = re.sub(r"^void ", "", r["kernel"])[:44]
    extra = ("%9.1f %5s %6.2f" % (r["floor_us"], r["bound"], r["frac_of_bound"])) if "floor_us" in r else ""
    print("%3d %-16s %-44s %9.1f %6.1f %s" % (r["pos"], r["wave"], kn, r["us"], 100.0 * r["us"] / total, extra))


if __name__ == "__main__":
  main()
