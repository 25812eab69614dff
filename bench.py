#!/usr/bin/env python
"""bench.py -- candidate-train examples/sec per AdaNet iteration (BASELINE.json metric).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]

A "step" is one training step of EVERY candidate of the iteration on one
minibatch (subnetwork fwd+bwd+update, candidate-ensemble head, EMA).  Workload
(config.workload): BASELINE configs[2] -- 8-candidate DNN search 100->H->H->10,
H in {64..1024}, 1M x 100 synthetic tabular data, B = 32768; it fits one GPU,
so N=1 trains all 8 candidates on one H100 and N>1 places the candidates on the GPUs
cost-balanced, training the ones heavier than a GPU's fair share (H=1024: 46 % of the step)
data-parallel on row slices of the minibatch over 2-4 GPUs (strong scaling: total work
fixed; the only data-path collective is one NCCL all-reduce of such a candidate's gradient
arena per step, captured in the step's CUDA graph; whole candidates exchange nothing until
the end-of-iteration loss all_gather).

Prints ONE JSON line on rank 0.  `value` = B*K / device time (CUDA events, max
over ranks) with the dataset resident in HBM; `e2e` = same metric through
the public adanet_b200.Estimator.train call with HOST (pinned) batches, H2D of every
batch and a D2H read of every step's losses (an `after_run` hook) inside the timed region.
`sustained` = the HBM-resident loop again for >= 2.5 s (power-capped steady state) with its own
clock samples; `roofline` carries the measured cuBLAS peak of the MMA kind the kernel issues
beside the bf16 peak of MEASURED_PEAKS.json (H100 SXM data sheet when absent); `cpu_baseline` = the faster of two
CPU restatements (NumPy/OpenBLAS oracle, torch-CPU oneDNN port) on the full B=32768 minibatch.

--dump-outputs DIR: the last timed step's losses and the iteration's trained state as float32 .npy (seeded inputs).
"""

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WIDTHS = (64, 128, 192, 256, 384, 512, 768, 1024)
IN_DIM, CLASSES, BATCH = 100, 10, 32768
DATA_ROWS = 1_000_000
METRIC = "candidate-train examples/sec per AdaNet iteration"
SUB_LR, ENS_LR, LAMBDA, BETA, DECAY = 0.05, 0.01, 0.01, 0.001, 0.9


def make_tabular(n, d=IN_DIM, classes=CLASSES, seed=1234):
  """SURVEY.md 8d synthetic tabular data: X ~ N(0,1) fp32 [n,d] (seed), teacher y = argmax(X@T + 0.5 eps),
  T ~ N(0,1) [d,classes] (seed+1), labels int64.  (Same construction as the oracle's generator; restated here so
  the product arm does not import test infrastructure.)"""
  rng = np.random.default_rng(seed)
  x = rng.standard_normal((n, d), dtype=np.float32)
  rng_t = np.random.default_rng(seed + 1)
  t = rng_t.standard_normal((d, classes), dtype=np.float32)
  eps = rng_t.standard_normal((n, classes), dtype=np.float32)
  y = np.argmax(x @ t + np.float32(0.5) * eps, axis=1).astype(np.int64)
  return x, y


def candidate_weights(iteration=0):
  """[(name, dims, complexity, ws, bs)] of the 8 candidates 100->H->H->10: glorot-uniform kernels from
  default_rng(1000 + 100*iteration + i), zero biases (SURVEY.md 8d), names as simple_dnn.py:124-131 de-duplicated."""
  out = []
  for i, h in enumerate(WIDTHS):
    dims = [IN_DIM, h, h, CLASSES]
    rng = np.random.default_rng(1000 + 100 * iteration + i)
    ws = []
    for a, b in zip(dims[:-1], dims[1:]):
      limit = np.sqrt(6.0 / (a + b))
      ws.append(rng.uniform(-limit, limit, size=(a, b)).astype(np.float32))
    bs = [np.zeros((b,), dtype=np.float32) for b in dims[1:]]
    name = "2_layer_dnn" if i == 0 else "2_layer_dnn_w%d" % h
    out.append((name, dims, float(np.sqrt(np.float32(2))), ws, bs))
  return out


def workload_name(gpus):
  how = ("all on one GPU" if gpus == 1 else
         "placed on %d GPUs cost-balanced, candidates heavier than a GPU's share row-sharded (data-parallel over 2-4 "
         "GPUs, one gradient all-reduce per step each)" % gpus)
  return ("configs[2]: 8-candidate DNN search 100->H->H->10, H in %s, 1Mx100 tabular synthetic, B=%d, candidates %s"
          % (list(WIDTHS), BATCH, how))


def train_flops_per_example():
  return sum(6 * (IN_DIM * h + h * h + h * CLASSES) - 2 * IN_DIM * h for h in WIDTHS)


class ClockSampler:
  """nvidia-smi clocks/throttle reasons DURING the timed region."""
  Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
       "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
       "clocks_event_reasons.sw_power_cap")

  def __init__(self, index=0):
    self.index, self.proc, self.lines = index, None, []

  def start(self):
    try:
      self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                    "--format=csv,noheader,nounits", "-lms", "50"],
                                   stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
      self.t = threading.Thread(target=self._read, daemon=True)
      self.t.start()
    except Exception:
      self.proc = None

  def _read(self):
    for line in self.proc.stdout:
      self.lines.append(line.strip())

  def stop(self):
    if not self.proc:
      return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
    self.proc.terminate()
    try:
      self.proc.wait(timeout=5)
    except Exception:
      self.proc.kill()
    sm, mx, reasons = [], [], set()
    names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
    for l in self.lines:
      f = [v.strip() for v in l.split(",")]
      if len(f) < 9:
        continue
      try:
        sm.append(float(f[1]))
        mx.append(float(f[2]))
      except ValueError:
        continue
      for n, v in zip(names, f[5:9]):
        if v.lower().startswith("active"):
          reasons.add(n)
    return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
            "reasons": sorted(reasons), "samples": len(sm)}


def load_peaks():   # fallback: H100 SXM data sheet (700 W), HBM3 3.35 TB/s, dense BF16 989 TFLOP/s
  p = os.path.join(ROOT, "MEASURED_PEAKS.json")
  if os.path.exists(p):
    with open(p) as f:
      d = json.load(f)
    return d.get("hbm_gbs", 3350.0), d.get("bf16_tflops", 989.0), d.get("bf16_tflops_sustained", 989.0), "measured"
  return 3350.0, 989.0, 989.0, "H100 SXM data sheet"


def _cpu_arms(cores):
  """The two CPU restatements of the reference's path on this box's host cores, each as (name, step_fn, threads):
  the NumPy/OpenBLAS oracle (oracle/adanet_oracle.py) and the torch-CPU (oneDNN/MKL) port (oracle/torch_cpu.py),
  both on the FULL B=32768 minibatch of the same 8-candidate workload.  bench.py's cpu_baseline / --impl reference
  legs are the only product-side places allowed to execute oracle/ code."""
  import torch
  from oracle import adanet_oracle as orc
  from oracle import torch_cpu
  x, y = make_tabular(BATCH * 2, seed=1234)
  cw = candidate_weights(0)
  arms = []
  # --- NumPy oracle
  o_specs = [orc.SubnetworkSpec(n, d, cx, ("sgd", SUB_LR), ws=[w.copy() for w in ws], bs=[b.copy() for b in bs])
             for n, d, cx, ws, bs in cw]
  ens = orc.EnsemblerSpec(optimizer=("sgd", ENS_LR), adanet_lambda=LAMBDA, adanet_beta=BETA)
  cands = orc.build_candidates(0, o_specs, [], ens, CLASSES, DECAY)
  it_np = [0]

  def step_numpy():
    off = (it_np[0] % 2) * BATCH
    orc.train_step(cands, [], ens, x[off:off + BATCH], y[off:off + BATCH])
    it_np[0] += 1

  arms.append(("numpy_openblas_oracle", step_numpy))
  # --- torch CPU port
  tc = [torch_cpu.Candidate(ws, bs, cx) for _, _, cx, ws, bs in cw]
  xt, yt = torch.tensor(x), torch.tensor(y)
  it_t = [0]

  def step_torch():
    off = (it_t[0] % 2) * BATCH
    torch_cpu.train_step(tc, xt[off:off + BATCH], yt[off:off + BATCH], SUB_LR, ENS_LR, LAMBDA, BETA, DECAY)
    it_t[0] += 1

  arms.append(("torch_cpu_onednn_port", step_torch))
  return arms


def _pick_cpu_arm(cores):
  """Times one step of each CPU arm at a few thread counts (NumPy/OpenBLAS is often fastest well below the core
  count; torch follows torch.set_num_threads) and returns the fastest (name, step_fn, threads, sweep)."""
  import torch
  try:
    from threadpoolctl import threadpool_limits
  except Exception:
    threadpool_limits = None
  arms = _cpu_arms(cores)
  # oversubscribed pools are slow on a many-core host (torch at 128 threads: 25 s per step on the bench box, 0.9 s at 16-32):
  # sweep at most 64 threads
  cand_threads = sorted({c for c in (min(cores, 64), 32, 16, 8) if 1 <= c <= cores}, reverse=True)
  sweep, best = {}, None
  for name, fn in arms:
    for th in cand_threads:
      if name.startswith("torch"):
        torch.set_num_threads(th)
        fn()
        t0 = time.perf_counter(); fn(); dt = time.perf_counter() - t0
      elif threadpool_limits is not None:
        with threadpool_limits(limits=th):
          fn()
          t0 = time.perf_counter(); fn(); dt = time.perf_counter() - t0
      else:
        if th != cores:
          continue
        fn()
        t0 = time.perf_counter(); fn(); dt = time.perf_counter() - t0
      sweep["%s@%d" % (name, th)] = round(dt, 3)
      if best is None or dt < best[3]:
        best = (name, fn, th, dt)
  name, fn, th, _ = best

  def run(n_steps):
    if name.startswith("torch"):
      torch.set_num_threads(th)
      t0 = time.perf_counter()
      for _ in range(n_steps):
        fn()
      return time.perf_counter() - t0
    ctx = threadpool_limits(limits=th) if threadpool_limits is not None else None
    if ctx is not None:
      ctx.__enter__()
    try:
      t0 = time.perf_counter()
      for _ in range(n_steps):
        fn()
      return time.perf_counter() - t0
    finally:
      if ctx is not None:
        ctx.__exit__(None, None, None)

  return name, run, th, sweep


def run_reference(args):
  """--impl reference: the reference's own implementation of the path is TF1 graph code on the TensorFlow CPU
  runtime (TensorFlow 2.1 is not installable here: Python 3.12, no network -- DESIGN.md section 2), so this arm
  times its CPU restatements on all host cores -- NumPy/OpenBLAS oracle and torch-CPU (oneDNN) port, the faster
  one -- on the SAME configuration as the GPU arm: 8 candidates, full B=32768 minibatches."""
  rank = int(os.environ.get("RANK", "0"))
  if rank != 0:
    return
  cores = os.cpu_count() or 1
  name, run, threads, sweep = _pick_cpu_arm(cores)
  run(max(1, min(args.warmup, 2)))
  steps = args.steps
  dt = run(steps)
  val = BATCH * steps / dt
  line = {
      "impl": "reference", "metric": METRIC, "value": val, "unit": "examples/s", "n_gpus": args.gpus,
      "steps": steps, "warmup": args.warmup, "ms_per_step": dt / steps * 1e3, "higher_is_better": True,
      "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
      "config": {"workload": workload_name(args.gpus), "candidates": len(WIDTHS), "batch": BATCH},
      "cpu_baseline": {"value": val, "unit": "examples/s", "cores": threads, "kind": "port", "arm": name,
                       "sample": "%d steps of the full B=%d minibatch of the same 8-candidate workload; fastest of "
                                 "{NumPy/OpenBLAS oracle, torch-CPU oneDNN port} x thread counts on %d host cores, "
                                 "seconds per step: %s (the TF1 reference itself is not installable: TensorFlow 2.1 "
                                 "absent)" % (steps, BATCH, cores, sweep)},
      "e2e": {"value": val, "unit": "examples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
  }
  print(json.dumps(line), flush=True)


def cpu_baseline_sample(seconds_budget=15.0):
  """The faster CPU restatement on all host cores, full-B steps for about `seconds_budget` seconds."""
  cores = os.cpu_count() or 1
  name, run, threads, sweep = _pick_cpu_arm(cores)
  per = min(sweep.values())
  n = int(max(2, min(200, seconds_budget / max(per, 1e-3))))
  dt = run(n)
  return {"value": BATCH * n / dt, "unit": "examples/s", "cores": threads, "kind": "port", "arm": name,
          "sample": "%d steps (%.1f s) of the full B=%d minibatch of the same 8-candidate workload; fastest of "
                    "{NumPy/OpenBLAS oracle, torch-CPU oneDNN port} x thread counts on %d host cores, s/step: %s"
                    % (n, dt, BATCH, cores, sweep)}


def measure_cublas_peaks(torch, n=8192, reps=10):
  """Dense tensor-core peaks of the MMA kinds this library issues, measured the way MEASURED_PEAKS.json measures
  bf16: cuBLAS matmul n^3, best of `reps`, CUDA events.  (cuBLAS is used for this yardstick only.)"""
  out = {}
  old = torch.backends.cuda.matmul.allow_tf32
  for kind in ("f16", "tf32"):
    try:
      if kind == "f16":
        a = torch.randn((n, n), device="cuda", dtype=torch.float16)
        b = torch.randn((n, n), device="cuda", dtype=torch.float16)
      else:
        torch.backends.cuda.matmul.allow_tf32 = True
        a = torch.randn((n, n), device="cuda")
        b = torch.randn((n, n), device="cuda")
      best = 1e9
      for i in range(reps + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); c = a @ b; e1.record(); e1.synchronize()
        if i >= 2:
          best = min(best, e0.elapsed_time(e1) * 1e-3)
      out[kind + "_tflops"] = 2.0 * n ** 3 / best / 1e12
      del a, b, c
    except Exception as exc:
      out[kind + "_tflops"] = None
      out[kind + "_error"] = repr(exc)
  torch.backends.cuda.matmul.allow_tf32 = old
  return out


def measure_dominant_kernel(lib, torch, reps=20):
  """CUDA-event timing of the dominant kernel of the step -- the H=1024 hidden-layer dense forward
  [32768,1024]x[1024,1024] + bias + ReLU, planes in / planes out, exactly as the engine launches it
  (adn_dense_fwd_p) -- on the stream it is launched on, L2 flushed between launches."""
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  B, I, O = BATCH, 1024, 1024
  sp = torch.cuda.current_stream()
  x = torch.randn((B, I), device="cuda")
  w = torch.randn((I, O), device="cuda") * 0.03
  b = torch.zeros((O,), device="cuda")
  xp, wp, yp = eng.new_planes(B, I, "cuda"), eng.new_planes(I, O, "cuda"), eng.new_planes(B, O, "cuda")
  _lib.check(lib.adn_planes_split(x.data_ptr(), B, I, xp.data_ptr(), sp.cuda_stream), "split")
  _lib.check(lib.adn_planes_split(w.data_ptr(), I, O, wp.data_ptr(), sp.cuda_stream), "split")
  flush = torch.empty((256 * 1024 * 1024 // 4,), device="cuda")   # 256 MB > 50 MB L2
  times = []
  for i in range(reps + 3):
    flush.fill_(float(i))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(sp)
    _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), b.data_ptr(), yp.data_ptr(), None, B, I, O, 1,
                                   sp.cuda_stream), "adn_dense_fwd_p")
    e1.record(sp)
    e1.synchronize()
    if i >= 3:
      times.append(e0.elapsed_time(e1) * 1e-3)
  f16 = _lib.plane_format() == _lib.PLANES_F16
  return float(np.mean(times)), 2.0 * B * I * O, "wgmma_3xf16_planes" if f16 else "mma_sync_3xtf32_planes"


def dump_outputs(dirpath, plan, limit_bytes=64 << 20, sample=1 << 21):
  """Last step's losses + trained state as float32 .npy; arrays over `sample` elements become a fixed, seeded sample."""
  os.makedirs(dirpath, exist_ok=True)
  arrays = {"last_losses": plan.last_losses()}
  for k, v in sorted(plan.state_dict().items()):
    if np.issubdtype(np.asarray(v).dtype, np.floating):
      arrays["state_" + k] = v
  for name, v in arrays.items():
    v = np.asarray(v, dtype=np.float32)
    if v.size > sample:
      arrays[name] = v.reshape(-1)[np.sort(np.random.default_rng(0).choice(v.size, size=sample, replace=False))]
    else:
      arrays[name] = v
  if sum(v.nbytes for v in arrays.values()) > limit_bytes:    # checked before anything is written
    raise RuntimeError("--dump-outputs: more than %d bytes" % limit_bytes)
  for name, v in arrays.items():
    np.save(os.path.join(dirpath, name + ".npy"), v)


def _finish(world):
  """Leaves a multi-rank job without tearing the NCCL communicators down one rank at a time: ranks other than 0 finish
  long before rank 0 (which still measures the roofline kernel and cuBLAS peaks), and destroying a sub-communicator
  (row-sharded candidates use process sub-groups) while a peer is still alive blocked the job until the launcher's
  timeout.  Everyone meets at a barrier once rank 0 has printed, then exits without the collective teardown."""
  if world <= 1:
    return
  import torch
  import torch.distributed as dist
  sys.stdout.flush()
  sys.stderr.flush()
  try:
    dist.barrier()
    torch.cuda.synchronize()
  finally:
    os._exit(0)


def run_ours(args):
  import torch
  import torch.distributed as dist
  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local = int(os.environ.get("LOCAL_RANK", "0"))
  torch.cuda.set_device(local)
  if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  from adanet_b200.distributed import exchange as ex
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  dev = torch.device("cuda", local)

  # Roofline of the dominant kernel, timed ALONE on a chip that has not yet been driven into its power cap -- the state
  # in which MEASURED_PEAKS.json's burst peak (its denominator) was taken -- together with the cuBLAS peaks of the MMA
  # kinds the library issues.  Rank 0 only; the other ranks wait at the first barrier.
  kt = kflops = kpath = peaks = None
  if rank == 0 and not args.profile:
    kt, kflops, kpath = measure_dominant_kernel(lib, torch)
    peaks = measure_cublas_peaks(torch)
    torch.cuda.synchronize()
    time.sleep(1.0)

  # synthetic data (SURVEY.md 8d), generated once on the host, replicated per GPU
  x_np, y_np = make_tabular(DATA_ROWS, IN_DIM, CLASSES, seed=1234)
  x_dev = torch.as_tensor(x_np).to(dev)
  y_dev = torch.as_tensor(y_np).to(dev)
  ens = eng.EnsemblerPlanSpec(optimizer=("sgd", ENS_LR), adanet_lambda=LAMBDA, adanet_beta=BETA)
  space = lambda t, frozen: [eng.SubnetworkPlanSpec(n, d, cx, ("sgd", SUB_LR), ws, bs, shared={"num_layers": 2})
                             for n, d, cx, ws, bs in candidate_weights(t)]

  # ---------------- value: dataset resident in HBM ----------------
  placement = "sharded" if world > 1 else "balanced"
  s = srch.AdaNetSearch(space, ens, IN_DIM, CLASSES, BATCH, device=dev, keep_traces=False, placement=placement)
  plan = s.build_iteration()
  batches = srch.consecutive_batches(x_dev, y_dev, BATCH)
  for _ in range(args.warmup):
    plan.train_step(*next(batches))
  torch.cuda.synchronize()
  if world > 1:
    dist.barrier()
  sampler = ClockSampler(local)
  if rank == 0:
    sampler.start()
  l0 = _lib.launch_count()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(args.steps):
    plan.train_step(*next(batches))
  e1.record()
  torch.cuda.synchronize()
  if world > 1:
    dist.barrier()
  secs = ex.max_over_ranks(e0.elapsed_time(e1) * 1e-3, device=dev)
  clocks = sampler.stop() if rank == 0 else None
  launches_local = plan.launches_per_step * args.steps if plan.launches_per_step else _lib.launch_count() - l0
  value = BATCH * args.steps / secs
  local_losses = plan.last_losses()
  assert np.isfinite(local_losses).all(), "non-finite loss in the timed region"
  if args.dump_outputs and rank == 0:
    dump_outputs(args.dump_outputs, plan)
  # ---------------- steady state: the same loop for >= 2.5 s (the chip reaches its power cap) ----------------
  sustained = None
  if not args.profile and args.sustain_seconds > 0:
    n_sus = int(min(20000, max(args.steps, args.sustain_seconds / max(secs / args.steps, 1e-5))))
    sampler2 = ClockSampler(local)
    if rank == 0:
      sampler2.start()
    torch.cuda.synchronize()
    if world > 1:
      dist.barrier()
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(n_sus):
      plan.train_step(*next(batches))
    s1.record()
    torch.cuda.synchronize()
    if world > 1:
      dist.barrier()
    sus_secs = ex.max_over_ranks(s0.elapsed_time(s1) * 1e-3, device=dev)
    sustained = {"steps": n_sus, "seconds": sus_secs, "ms_per_step": sus_secs / n_sus * 1e3,
                 "value": BATCH * n_sus / sus_secs, "unit": "examples/s",
                 "clocks": sampler2.stop() if rank == 0 else None}
    assert np.isfinite(plan.last_losses()).all(), "non-finite loss in the sustained region"
  rep = s.finish_iteration(secs)   # end-of-iteration all_gather + selection (outside the timed region)
  if args.profile:   # under ncu: only the in-HBM step loop (a number printed under a profiler is never a bench value)
    if rank == 0:
      print(json.dumps({"profile_only": True, "ms_per_step_under_profiler": secs / args.steps * 1e3,
                        "gpu_launches": int(launches_local)}), flush=True)
    _finish(world)
    return

  # ---------------- e2e: host batches through the PUBLIC API (adanet.Estimator.train) ----------------
  e2e_steps = min(args.steps, 100)
  n_host = BATCH * 4
  x_host = torch.as_tensor(x_np[:n_host]).pin_memory()
  y_host = torch.as_tensor(y_np[:n_host]).pin_memory()
  warm = max(3, args.warmup)

  def host_batches(n):
    def fn():
      for i in range(n):
        o = (i % 4) * BATCH
        yield {"x": x_host[o:o + BATCH]}, y_host[o:o + BATCH]
    return fn

  e2e_api, e2e_note, e2e_secs, d2h = "adanet_b200.Estimator.train", None, None, 0
  try:
    import adanet_b200 as adanet
    from adanet_b200 import graph, train

    class _WidthBuilder(adanet.subnetwork.Builder):
      """100 -> H -> H -> 10 with the same injected weights as the device-resident run."""

      def __init__(self, spec):
        self._spec = spec

      name = property(lambda self: self._spec.name)

      def build_subnetwork(self, features, logits_dimension, training, iteration_step, summary, previous_ensemble=None):
        h = graph.input_layer(features, [graph.numeric_column("x", IN_DIM)])
        n = len(self._spec.ws)
        for i, (w, b) in enumerate(zip(self._spec.ws, self._spec.bs)):
          h = graph.dense(h, w.shape[1], activation=graph.relu if i < n - 1 else None,
                          kernel_initializer=graph.constant_initializer(w), bias_initializer=graph.constant_initializer(b))
          if i == n - 2:
            last = h
        return adanet.Subnetwork(last_layer=last, logits=h, complexity=self._spec.complexity)

      def build_subnetwork_train_op(self, subnetwork, loss, var_list, labels, iteration_step, summary, previous_ensemble):
        return train.GradientDescentOptimizer(SUB_LR).minimize(loss=loss, var_list=var_list)

    class _Losses:
      last = None

      def after_run(self, run_context, run_values):      # D2H read of every step's losses
        self.last = run_values.results["losses"]

    import tempfile
    # a multi-rank Estimator needs a model_dir like the reference's (estimator.py:632-644); only the chief writes to it
    model_dir = None
    if world > 1:        # a fresh directory, chosen by rank 0, so that nothing of an earlier run can be restored from it
      box = [tempfile.mkdtemp(prefix="adanet_b200_bench_") if rank == 0 else None]
      dist.broadcast_object_list(box, src=0)
      model_dir = box[0]
    est = adanet.Estimator(
        model_dir=model_dir,
        head=adanet.heads.MultiClassHead(CLASSES),
        subnetwork_generator=adanet.subnetwork.SimpleGenerator([_WidthBuilder(sp) for sp in space(0, [])]),
        max_iteration_steps=10 ** 9, max_iterations=1, candidate_placement=placement,
        ensemblers=[adanet.ensemble.ComplexityRegularizedEnsembler(optimizer=train.GradientDescentOptimizer(ENS_LR),
                                                                   adanet_lambda=LAMBDA, adanet_beta=BETA)])
    hook = _Losses()
    est.train(host_batches(warm), steps=warm, hooks=[hook])          # builds the plan, captures the graph
    torch.cuda.synchronize()
    if world > 1:
      dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    # every step: host->device copy of its (pinned) minibatch, started under the previous step's kernels, and a
    # device->host read of its losses through the hook
    est.train(host_batches(e2e_steps), steps=e2e_steps, hooks=[hook])
    e1.record()
    torch.cuda.synchronize()
    e2e_secs = e0.elapsed_time(e1) * 1e-3
    d2h = int(hook.last.nbytes)
  except Exception as exc:      # measured below through the engine-level search API instead; the reason is reported
    e2e_api, e2e_note = "adanet_b200.core.search.AdaNetSearch.train_iteration", "Estimator path not used: %r" % (exc,)
    s2 = srch.AdaNetSearch(space, ens, IN_DIM, CLASSES, BATCH, device=dev, keep_traces=False, placement=placement)
    plan2 = s2.build_iteration()
    hb = srch.consecutive_batches(x_host, y_host, BATCH)
    for _ in range(warm):
      plan2.train_step(*next(hb))
      plan2.last_losses()
    torch.cuda.synchronize()
    host_losses = None

    def read_losses(plan):
      nonlocal host_losses
      host_losses = plan.last_losses()

    e2e_secs = s2.train_iteration(hb, e2e_steps, on_step=read_losses)
    torch.cuda.synchronize()
    d2h = int(host_losses.nbytes)
  if world > 1:
    dist.barrier()
  e2e_secs = ex.max_over_ranks(e2e_secs, device=dev)
  e2e = {"value": BATCH * e2e_steps / e2e_secs, "unit": "examples/s",
         "h2d_bytes_per_step": BATCH * IN_DIM * 4 + BATCH * 8, "d2h_bytes_per_step": d2h, "steps": e2e_steps,
         "api": e2e_api}
  if e2e_note:
    e2e["note"] = e2e_note

  if rank != 0:
    _finish(world)
    return

  # ---------------- roofline of the dominant kernel + CPU baseline (rank 0, N=1 only for cpu) ----------------
  hbm, bf16_burst, bf16_sust, which = load_peaks()
  achieved = kflops / kt / 1e12
  f16 = kpath.startswith("wgmma_3xf16")
  kind_peak = peaks.get("f16_tflops" if f16 else "tf32_tflops")
  plane_bytes = 2 * (2 if f16 else 4)      # hi + lo bytes per value
  roofline = {
      "bound": "tensor", "kernel": "adn_dense_fwd_p [32768,1024]x[1024,1024] bias+relu, planes in/out (%s)" % kpath,
      "achieved": achieved, "peak": bf16_burst, "unit": "TFLOP/s", "frac": achieved / bf16_burst,
      "peak_source": "bf16 peak (%s); numerator = algorithmic fp32 FLOPs 2*B*in*out; the tensor-core "
                     "path issues 3 MMAs per product (hi*hi, hi*lo, lo*hi split for 1e-5 fp32 parity), so the design "
                     "ceiling of `frac` is 1/3 with fp16 planes (1/6 with the TF32 fallback)" % which,
      "mma_kind": "wgmma f16" if f16 else "mma.sync tf32", "mmas_per_product": 3,
      "kind_peak_measured_tflops": kind_peak, "kind_peaks_measured": peaks,
      "issued_frac_of_kind_peak": (3.0 * achieved / kind_peak) if kind_peak else None,
      "useful_frac_of_kind_peak": (achieved / kind_peak) if kind_peak else None,
      "traffic_unit": "algorithmic: %.1f MB of split planes (%d B/value) = %.1f MB of "
                      "the fp32 tensors they represent" % ((2 * BATCH * 1024 + 1024 * 1024) * plane_bytes / 1e6, plane_bytes,
                                                           (2 * BATCH * 1024 + 1024 * 1024) * 4 / 1e6),
      "launch_seconds": kt,
  }
  cpu = cpu_baseline_sample() if world == 1 else None
  line = {
      "metric": METRIC, "value": value, "unit": "examples/s", "n_gpus": world, "steps": args.steps,
      "warmup": args.warmup, "ms_per_step": secs / args.steps * 1e3, "higher_is_better": True, "scaling": "strong",
      "vs_baseline": None, "dtype": "f32", "data": "synthetic",
      "config": {"workload": workload_name(world), "candidates": len(WIDTHS), "batch": BATCH,
                 "l2_policy": "inputs larger than L2: every step reads a fresh 32768x100 slice of the 400 MB "
                              "HBM-resident dataset and streams >1 GB of activations; weights stay cache-resident "
                              "as in real training",
                 "train_flops_per_example": train_flops_per_example(),
                 "candidate_examples_per_sec": value * len(WIDTHS),
                 "cuda_graph": True, "selected": rep.candidate_names[rep.best_index]},
      "clocks": clocks, "e2e": e2e, "gpu_launches": int(launches_local),
      "roofline": roofline, "cpu_baseline": cpu, "sustained": sustained,
      "plane_format": "f16" if _lib.plane_format() == _lib.PLANES_F16 else "tf32",
      "useful_tflops": value * train_flops_per_example() / 1e12,
  }
  print(json.dumps(line), flush=True)
  _finish(world)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--gpus", type=int, default=1)
  ap.add_argument("--steps", type=int, default=200)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
  ap.add_argument("--profile", action="store_true", help="step loop only (for ncu captures)")
  ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                  help="write the last timed step's losses and trained state to DIR/<name>.npy (float32); with N > 1 "
                       "GPUs, those of the candidates rank 0 trains")
  ap.add_argument("--sustain-seconds", type=float, default=2.5,
                  help="length of the additional steady-state measurement (0 = skip)")
  args = ap.parse_args()
  if args.impl == "reference":
    run_reference(args)
  else:
    run_ours(args)


if __name__ == "__main__":
  main()
