"""Wide head kernel (adn_head_group_wide) measurements, one JSON line per result:

  1. the wide head group alone at B = 32768, C in {100, 1000}, N in {1, 2, 4, 8}, SCALAR and VECTOR mixture weights with
     grads, dens and planes: us per call (CUDA events over many launches after warm-up), algorithmic bytes (members read
     once, labels, dens and both planes written), GB/s and the fraction of the H100 SXM's 3.35 TB/s;
  2. narrow (adn_head_group) against wide at shapes both run, C in {10, 64}, alternated;
  3. one training step of the configs[2] candidates (8 nets 100->H->H->C, B = 32768) for C in {10, 100, 1000}: ms per
     step (CUDA-graph replays) and launches per step.

The card's name and power limit are read in the same run and printed first."""

import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except Exception as e:   # noqa: BLE001
    out = "nvidia-smi unavailable: %s" % e
  return out


def time_us(torch, fn, reps=50, warm=5):
  for _ in range(warm):
    fn()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record()
  for _ in range(reps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) * 1e3 / reps


def head_call(torch, lib, _lib, B, C, N, mix, wide, planes=True):
  dev = torch.device("cuda")
  members = [torch.randn((B, C), device=dev) for _ in range(N)]
  labels = torch.randint(0, C, (B,), device=dev)
  w = torch.full((N,) if mix == _lib.MIX_SCALAR else (N, C), 1.0 / N, device=dev)
  dw, dbias, out3 = torch.empty_like(w), torch.empty(C, device=dev), torch.empty(3, device=dev)
  dens = torch.empty((B, C), device=dev)
  pl = torch.zeros(_lib.query(_lib.Q_PLANES_BYTES, B, C), dtype=torch.uint8, device=dev) if planes else None
  ws = torch.empty(_lib.query(_lib.Q_HEAD_WIDE_WS if wide else _lib.Q_HEAD_WS, B, C, N), dtype=torch.uint8, device=dev)
  mp = _lib.ptr_array([m.data_ptr() for m in members])
  gam = _lib.f32_array([0.001] * N)
  op = _lib.HeadOp(0, mix, ctypes.cast(mp, ctypes.POINTER(ctypes.c_void_p)), N, 0, w.data_ptr(), None,
                   ctypes.cast(gam, ctypes.POINTER(ctypes.c_float)), 2.0, 0, labels.data_ptr(), None, out3.data_ptr(),
                   dw.data_ptr(), dbias.data_ptr(), dens.data_ptr(), None, pl.data_ptr() if planes else None, 0, 0,
                   ws.data_ptr(), ws.numel())
  arr = (_lib.HeadOp * 1)(op)
  f = lib.adn_head_group_wide if wide else lib.adn_head_group
  keep = (members, labels, w, dw, dbias, out3, dens, pl, ws, mp, gam, arr)
  esize = 2 if _lib.plane_format() == _lib.PLANES_F16 else 4
  nbytes = N * B * C * 4 + B * 8 + B * C * 4 + (2 * B * C * esize if planes else 0)
  return (lambda: _lib.check(f(arr, 1, B, C, None), "head")), nbytes, keep


def step_bench(torch, C, steps=20, warm=3):
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  widths, B, D = (64, 128, 192, 256, 384, 512, 768, 1024), 32768, 100

  def space(t, frozen):
    out = []
    for i, h in enumerate(widths):
      dims = [D, h, h, C]
      rng = np.random.default_rng(1000 + 100 * t + i)
      ws = [rng.uniform(-np.sqrt(6.0 / (a + b)), np.sqrt(6.0 / (a + b)), size=(a, b)).astype(np.float32)
            for a, b in zip(dims[:-1], dims[1:])]
      bs = [np.zeros((b,), np.float32) for b in dims[1:]]
      out.append(eng.SubnetworkPlanSpec("2_layer_dnn_w%d" % h, dims, float(np.sqrt(2.0)), ("sgd", 0.05), ws, bs,
                                        shared={"num_layers": 2}))
    return out

  dev = torch.device("cuda")
  rng = np.random.default_rng(1234)
  x = torch.as_tensor(rng.standard_normal((B * 4, D), dtype=np.float32)).to(dev)
  y = torch.as_tensor(rng.integers(0, C, B * 4)).to(dev)
  ens = eng.EnsemblerPlanSpec(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001)
  s = srch.AdaNetSearch(space, ens, D, C, B, device=dev, keep_traces=False)
  plan = s.build_iteration()
  batches = srch.consecutive_batches(x, y, B)
  for _ in range(warm):
    plan.train_step(*next(batches))
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(steps):
    plan.train_step(*next(batches))
  e1.record()
  torch.cuda.synchronize()
  return dict(kind="step", C=C, ms_per_step=e0.elapsed_time(e1) / steps, launches_per_step=plan.launches_per_step,
              head_path=_lib.query(_lib.Q_HEAD_PATH, C, 1))


def main():
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  print(json.dumps({"card": card(), "plane_format": _lib.plane_format()}), flush=True)
  # 1. wide head alone
  for C in (100, 1000):
    for N in (1, 2, 4, 8):
      for mix, mname in ((_lib.MIX_SCALAR, "scalar"), (_lib.MIX_VECTOR, "vector")):
        fn, nbytes, keep = head_call(torch, lib, _lib, 32768, C, N, mix, True)
        us = time_us(torch, fn)
        print(json.dumps(dict(kind="wide", B=32768, C=C, N=N, mix=mname, us=round(us, 2), bytes=nbytes,
                              gbs=round(nbytes / us / 1e3, 1), frac_hbm=round(nbytes / (us * 1e-6) / HBM, 3))), flush=True)
        del keep
  # 2. narrow vs wide, alternated
  for C, N in ((10, 1), (10, 8), (64, 1), (64, 4)):
    fa, nbytes, ka = head_call(torch, lib, _lib, 32768, C, N, _lib.MIX_SCALAR, False)
    fb, _, kb = head_call(torch, lib, _lib, 32768, C, N, _lib.MIX_SCALAR, True)
    ta, tb = [], []
    for _ in range(5):
      ta.append(time_us(torch, fa))
      tb.append(time_us(torch, fb))
    print(json.dumps(dict(kind="narrow_vs_wide", B=32768, C=C, N=N, narrow_us=[round(t, 2) for t in ta],
                          wide_us=[round(t, 2) for t in tb], bytes=nbytes)), flush=True)
    del ka, kb
  # 3. training steps of the configs[2] candidates
  for C in (10, 100, 1000):
    print(json.dumps(step_bench(torch, C)), flush=True)


if __name__ == "__main__":
  main()
