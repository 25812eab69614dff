"""Device time of the benchmark's two thin-K plane GEMM waves, each launched alone (one GPU).

  python tools/bench_thin_k.py [--reps 200]

The waves of bench.py's training step (batch 32768, the 8 candidate widths): the first-layer forward (K = 100, planes
out with bias and ReLU) and the logits layer's dX (K = 10, planes out with the ReLU mask and column sums).  Each is one
grouped call (dX with its column-sum reduction launch), timed with CUDA events over --reps back-to-back calls after a warm-up; the card's name, power limit and
clocks are read in the same run.  Floors are step_profile.gemm_waves' algorithmic HBM bytes over the data-sheet 3.35 TB/s.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.step_profile import gemm_waves  # noqa: E402

HBM = 3.35e12


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=200)
  args = ap.parse_args()
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  _lib.set_plane_format(_lib.PLANES_F16)
  B, I, C, widths = bench.BATCH, bench.IN_DIM, bench.CLASSES, bench.WIDTHS
  st = torch.cuda.current_stream().cuda_stream
  rng = np.random.default_rng(7)

  def planes(a, log2_scale=0):
    r, c = a.shape
    pl = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, r, c) // 4,), device="cuda")
    src = torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    _lib.check(lib.adn_planes_split_scaled(src.data_ptr(), r, c, pl.data_ptr(), log2_scale, st), "split")
    return pl

  keep = []
  xp = planes(rng.standard_normal((B, I)))
  fops = []
  for h in widths:
    wp, b = planes(rng.standard_normal((I, h)) / np.sqrt(I)), torch.randn(h, device="cuda")
    yp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, h) // 4,), device="cuda")
    keep += [wp, b, yp]
    fops.append(_lib.FwdOp(xp.data_ptr(), wp.data_ptr(), b.data_ptr(), yp.data_ptr(), None, I, h, _lib.ACT_RELU, 0))
  dzp = planes(rng.standard_normal((B, C)), 7)
  bops = []
  for h, yp in zip(widths, keep[2::3]):
    wp = planes(rng.standard_normal((h, C)) / np.sqrt(C))
    dxp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, h) // 4,), device="cuda")
    cs = torch.zeros(h, device="cuda")
    ws_bytes = _lib.query(_lib.Q_DENSE_BWD_P_WS, B, h, C)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device="cuda")
    keep += [wp, dxp, cs, ws]
    bops.append(_lib.BwdOp(yp.data_ptr(), wp.data_ptr(), dzp.data_ptr(), dxp.data_ptr(), None, cs.data_ptr(), None, h, C,
                           1, 7, ws.data_ptr(), ws_bytes, 0.0, 0.0))
  fa, ba = (_lib.FwdOp * len(fops))(*fops), (_lib.BwdOp * len(bops))(*bops)
  nbytes = {w[0]: w[3] for w in gemm_waves()}
  waves = {"fwd L1": lambda: lib.adn_dense_fwd_p_group(fa, len(fops), B, st),
           "bwd k=0 dX": lambda: lib.adn_dense_bwd_p_group(ba, len(bops), B, st)}
  info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                        capture_output=True, text=True).stdout.strip()
  print("GPU:", info)
  for name, fn in waves.items():
    for _ in range(10):
      _lib.check(fn(), name)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.reps):
      fn()
    t1.record()
    torch.cuda.synchronize()
    us = t0.elapsed_time(t1) * 1e3 / args.reps
    floor = nbytes[name] / HBM * 1e6
    print("%-11s %8.1f us per group call  HBM floor %6.1f us  frac %.2f" % (name, us, floor, floor / us))
  print("GPU after:", subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True).stdout.strip())


if __name__ == "__main__":
  main()
