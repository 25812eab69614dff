#!/usr/bin/env python
"""CUDA-event timing of the multi-source forward of the grouped plane GEMM (adn_fwd_op.srcs) against the
single-source GEMM of the same M, N and total K over the materialised concatenation, in the current plane format.

Each figure is printed with its fraction of the hardware floor: the larger of the tensor-core time (three products
per multiply-add, hi*hi + hi*lo + lo*hi, at the data-sheet dense FP16 or TF32 rate) and the HBM time (operand and
output planes read or written once, at 3.35 TB/s).  The card's name and power limit are read in the same run.

  python tools/bench_connections.py [--iters 200] [--tf32]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12
PEAK_FLOPS = {"f16": 989e12, "tf32": 495e12}       # H100 SXM data sheet, dense, 700 W
# (batch, piece widths, out): the flagship hidden width reading one frozen hidden layer of the same width, and a
# narrow layer of K = 896 cut into 1..4 pieces of whole k-blocks, so that the cost of a piece boundary shows apart
# from K (one piece is the single-source kernel)
SHAPES = [(32768, [1024, 1024], 1024), (32768, [448, 448], 256), (32768, [256, 512, 128], 256),
          (32768, [128, 256, 256, 256], 256)]


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return out
  except (OSError, subprocess.CalledProcessError, IndexError):
    return "unknown"


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--iters", type=int, default=200)
  ap.add_argument("--tf32", action="store_true")
  args = ap.parse_args()
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  if not torch.cuda.is_available():
    raise SystemExit("bench_connections: no GPU")
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  fmt = "tf32" if args.tf32 else "f16"
  _lib.set_plane_format(_lib.PLANES_TF32 if args.tf32 else _lib.PLANES_F16)
  esize = 4 if args.tf32 else 2
  stream = torch.cuda.current_stream().cuda_stream
  planes = lambda r, c: torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, r, c) // 4,), device="cuda")

  def split(a):
    p = planes(*a.shape)
    _lib.check(lib.adn_planes_split(a.data_ptr(), a.shape[0], a.shape[1], p.data_ptr(), stream), "split")
    return p

  def timed(fn):
    for _ in range(10):
      fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
      fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / args.iters

  results = []
  gen = torch.Generator(device="cuda").manual_seed(0)
  for B, widths, N in SHAPES:
    K = sum(widths)
    xs = [torch.randn(B, w, device="cuda", generator=gen) for w in widths]
    ws = [torch.randn(w, N, device="cuda", generator=gen) / K ** 0.5 for w in widths]
    bias = torch.zeros(N, device="cuda")
    xps, wps = [split(x) for x in xs], [split(w) for w in ws]
    xcat, wcat = split(torch.cat(xs, 1)), split(torch.cat(ws, 0))
    y_ms, y_ss = planes(B, N), planes(B, N)
    srcs = (_lib.FwdSrc * (len(widths) - 1))(*[_lib.FwdSrc(x.data_ptr(), w.data_ptr(), n)
                                               for x, w, n in zip(xps[1:], wps[1:], widths[1:])])
    ms = _lib.FwdOp(xps[0].data_ptr(), wps[0].data_ptr(), bias.data_ptr(), y_ms.data_ptr(), None, widths[0], N,
                    _lib.ACT_RELU, 0)
    ms.srcs, ms.n_srcs = ctypes.cast(srcs, ctypes.POINTER(_lib.FwdSrc)), len(widths) - 1
    ss = _lib.FwdOp(xcat.data_ptr(), wcat.data_ptr(), bias.data_ptr(), y_ss.data_ptr(), None, K, N, _lib.ACT_RELU, 0)
    ms_arr, ss_arr = (_lib.FwdOp * 1)(ms), (_lib.FwdOp * 1)(ss)
    run_ms = lambda: _lib.check(lib.adn_dense_fwd_p_group(ms_arr, 1, B, stream), "multi-source fwd")
    run_ss = lambda: _lib.check(lib.adn_dense_fwd_p_group(ss_arr, 1, B, stream), "single-source fwd")
    t_ms = t_ss = float("inf")
    for _ in range(3):                     # alternated, best of three: the two see the same clocks
      t_ms, t_ss = min(t_ms, timed(run_ms)), min(t_ss, timed(run_ss))
    flops = 3 * 2.0 * B * N * K
    nbytes = 2 * esize * (B * K + K * N + B * N)
    floor = max(flops / PEAK_FLOPS[fmt], nbytes / HBM_BPS)
    bound = "tensor" if flops / PEAK_FLOPS[fmt] >= nbytes / HBM_BPS else "hbm"
    for name, t in (("multi_source", t_ms), ("single_source_concat", t_ss)):
      results.append({"shape": {"batch": B, "pieces": widths, "out": N}, "kernel": name, "format": fmt,
                      "us": round(t * 1e6, 2), "floor_us": round(floor * 1e6, 2), "floor_bound": bound,
                      "fraction_of_floor": round(floor / t, 3)})
  print(json.dumps({"card": card(), "iters": args.iters, "results": results}, indent=1))


if __name__ == "__main__":
  main()
