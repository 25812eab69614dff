"""Which plane GEMM kernels (csrc/planes.cu) a call launches, read from torch.profiler: the kernel-choice checks of
test_gpu_thin_k, test_gpu_dw_wide and test_gpu_wide_fwd.

Profiling a whole training step left later profiler sessions of the same process without CUDA events, so the checks
that profile one run it in a child process (in_child).
"""

import json
import os
import subprocess
import sys

KERNELS = ("pl_gemm_kernel", "pl_gemm_ms_kernel", "pl_thin_kernel", "pl_dw_kernel", "pl_wide_kernel")


def kernels(torch, fn):
  """short names (pl_gemm_kernel<1, 0>, pl_thin_kernel<0>, pl_dw_kernel, ...) of the plane GEMM kernels fn launches,
  in order"""
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  out = []
  for e in prof.events():
    if e.device_type.name != "CUDA":
      continue
    for k in KERNELS:
      i = e.name.find(k)
      if i >= 0:
        rest = e.name[i + len(k):]
        out.append(k + rest.split(">")[0] + ">" if rest.startswith("<") else k)
        break
  return out


def bench_step_kernels():
  """kernel names of one eager training step of bench.py's workload (8 candidates 100 -> H -> H -> 10, B = 32768)"""
  from tests.test_gpu_plane_groups import _open
  torch, _, _ = _open()
  import bench
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  dev = torch.device("cuda", 0)
  x_np, y_np = bench.make_tabular(2 * bench.BATCH, bench.IN_DIM, bench.CLASSES, seed=1234)
  x_dev, y_dev = torch.as_tensor(x_np).to(dev), torch.as_tensor(y_np).to(dev)
  ens = eng.EnsemblerPlanSpec(optimizer=("sgd", bench.ENS_LR), adanet_lambda=bench.LAMBDA, adanet_beta=bench.BETA)
  space = lambda t, frozen: [eng.SubnetworkPlanSpec(n, d, cx, ("sgd", bench.SUB_LR), ws, bs, shared={"num_layers": 2})
                             for n, d, cx, ws, bs in bench.candidate_weights(t)]
  s = srch.AdaNetSearch(space, ens, bench.IN_DIM, bench.CLASSES, bench.BATCH, device=dev, keep_traces=False,
                        placement="balanced")
  plan = s.build_iteration()
  plan.use_cuda_graph = False
  batches = srch.consecutive_batches(x_dev, y_dev, bench.BATCH)
  plan.train_step(*next(batches))
  return kernels(torch, lambda: plan.train_step(*next(batches)))


def in_child(module, fn):
  """runs tests.<module>.<fn>() in a fresh interpreter started like this one and returns its result (JSON)"""
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  flags = [f for f, on in (("-I", sys.flags.isolated), ("-E", sys.flags.ignore_environment),
                           ("-s", sys.flags.no_user_site)) if on]
  code = ("import json, sys; sys.path.insert(0, %r); from tests import %s as t; "
          "print('RESULT ' + json.dumps(t.%s()))" % (root, module, fn))
  r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=root, capture_output=True, text=True, timeout=900)
  lines = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
  assert r.returncode == 0 and lines, "child process failed (%d):\n%s\n%s" % (r.returncode, r.stdout[-3000:],
                                                                         r.stderr[-3000:])
  return json.loads(lines[-1][len("RESULT "):])
