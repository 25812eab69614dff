"""GPU probe (not a pytest test): componentwise error of the dense paths vs float64.

  python tests/probe_accuracy.py

On the inputs of the non-cancelling and wide-range tests in tests/test_gpu_plane_groups.py (all-positive forward
at K = 4096, all-positive split-K dW at K = batch = 32768 with dz carried as dz * 2^15, rows scaled by 2^-8 .. 2^8),
prints for the plane path in both formats (fp16 and TF32 planes) and, as a baseline, the fp32 SIMT path:
max |err| / (|A| |B|)_ij, the quantity those tests bound by 3e-6, and the signed mean of err / (|A| |B|)_ij, which
shows a rounding bias.
"""

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _report(label, path, got, exact, scale):
  r = (got.astype(np.float64) - exact) / scale
  print("%-34s %-5s max err/|A||B| = %.3e   mean = % .3e" % (label, path, np.abs(r).max(), r.mean()), flush=True)


def main():
  import torch
  from tests import test_gpu_plane_groups as t
  _, _lib, lib = t._open()
  sp = torch.cuda.current_stream().cuda_stream
  before = _lib.plane_format()

  def planes(a, s=0):
    return t._planes(torch, _lib, lib, a, s)

  def plane_fwd(x, w):
    (B, I), O = x.shape, w.shape[1]
    y = torch.empty((B, O), device="cuda")
    xp, wp = planes(x), planes(w)
    _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, None, y.data_ptr(), B, I, O, 0, sp), "fwd_p")
    return y.cpu().numpy()

  def plane_dw(x, dz, s):
    (B, I), O = x.shape, dz.shape[1]
    nb = _lib.query(_lib.Q_DENSE_BWD_P_WS, B, I, O)
    ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")
    dw = torch.empty((I, O), device="cuda")
    xp, dzp = planes(x), planes(dz, s)
    _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), None, dzp.data_ptr(), None, None, None, dw.data_ptr(), B, I, O, 0, s,
                                   ws.data_ptr(), nb, sp), "bwd_p")
    return dw.cpu().numpy()

  def simt_fwd(x, w):
    (B, I), O = x.shape, w.shape[1]
    y = torch.empty((B, O), device="cuda")
    xd, wd = torch.as_tensor(x).cuda(), torch.as_tensor(w).cuda()
    _lib.check(lib.adn_dense_fwd(xd.data_ptr(), wd.data_ptr(), None, y.data_ptr(), B, I, O, 0, None, 0, sp), "fwd")
    return y.cpu().numpy()

  def simt_dw(x, dz):
    (B, I), O = x.shape, dz.shape[1]
    nb = _lib.query(_lib.Q_DENSE_BWD_WS, B, I, O)
    ws = torch.empty((max(nb, 16),), dtype=torch.uint8, device="cuda")
    xd, dzd = torch.as_tensor(x).cuda(), torch.as_tensor(dz).cuda()
    dw, db = torch.empty((I, O), device="cuda"), torch.empty((O,), device="cuda")
    _lib.check(lib.adn_dense_bwd(xd.data_ptr(), None, dzd.data_ptr(), None, dw.data_ptr(), db.data_ptr(), B, I, O, 0,
                                 ws.data_ptr(), nb, sp), "bwd")
    return dw.cpu().numpy()

  xf, wf = t.positive_fwd_inputs()
  xd, dzd, s = t.positive_dw_inputs()
  xr, wr, _ = t.row_spread_inputs()
  cases = []
  for label, a, b in (("all-positive fwd  K=4096", xf, wf), ("row-spread fwd    K=1024", xr, wr)):
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    cases.append((label, "fwd", (a, b), a64 @ b64, np.abs(a64) @ np.abs(b64)))
  a64, b64 = xd.astype(np.float64), dzd.astype(np.float64)
  cases.append(("all-positive dW    K=32768", "dw", (xd, dzd), a64.T @ b64, np.abs(a64).T @ np.abs(b64)))
  try:
    for label, kind, args, exact, scale in cases:
      for name, fmt in (("f16", _lib.PLANES_F16), ("tf32", _lib.PLANES_TF32)):
        _lib.set_plane_format(fmt)
        got = plane_fwd(*args) if kind == "fwd" else plane_dw(*args, s)
        _report(label, name, got, exact, scale)
      _lib.set_dense_path(_lib.PATH_SIMT)
      got = simt_fwd(*args) if kind == "fwd" else simt_dw(*args)
      _report(label, "simt", got, exact, scale)
      _lib.set_dense_path(_lib.PATH_AUTO)
  finally:
    _lib.set_plane_format(before)
    _lib.set_dense_path(_lib.PATH_AUTO)


if __name__ == "__main__":
  main()
