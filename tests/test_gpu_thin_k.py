"""The thin-K plane GEMM (csrc/planes.cu pl_thin_kernel): groups whose every problem is one fp16 accumulation chunk
(K <= 128) with planes out run on it, every other group on pl_gemm_kernel.

Each op runs alone (thin kernel) and in one call with a K = 257 op (the group then takes pl_gemm_kernel); the two
results must agree byte for byte -- hi and lo' planes, sign-bit words, the per-32-row column sums and their reduction
-- and each is checked against float64 with the componentwise bounds of test_gpu_plane_groups.
"""

import numpy as np
import pytest

from tests.plane_kernels import kernels as _kernels
from tests.test_gpu_plane_groups import (DX_MUL, _bwd_case, _bwd_check, _bwd_run, _bytes_equal, _fwd_case, _fwd_check,
                                         _fwd_run, _fwd_struct, _open, _stream)

pytestmark = pytest.mark.gpu

# forward ops (in, out, bias, act, planes out, dropout): K in {1, 10, 64, 65, 100, 128}, N in {10, 33, 64, 200, 1024};
# the last op (K = 257) is the partner that sends a group to pl_gemm_kernel
FWD_OPS = [
    (1, 10, 1, 1, 1, None),
    (10, 33, 0, 0, 1, None),
    (64, 64, 1, 1, 1, (5, 0)),
    (65, 200, 1, 0, 1, None),
    (100, 1024, 1, 1, 1, (6, 1)),
    (128, 33, 0, 1, 1, None),
    (100, 200, 1, 1, 1, None),
    (10, 1024, 0, 0, 1, None),
    (257, 64, 1, 1, 1, None),
]
# backward ops (in, out, x_relu_mask, dz_log2_scale, dx_mul, outputs): dX has K = out; masks on 33 and 200 columns
# clip the last 32-column block
BWD_OPS = [
    (33, 10, 1, 7, 0.0, "dxp cs"),
    (200, 1, 1, 0, DX_MUL, "dxp cs"),
    (64, 64, 0, 15, DX_MUL, "dxp"),
    (1024, 100, 1, 7, 0.0, "dxp cs"),
    (10, 128, 0, 0, 0.0, "dxp cs"),
    (200, 65, 1, 15, DX_MUL, "dxp"),
    (100, 257, 1, 7, 0.0, "dxp cs"),
]
BATCHES = [1, 129, 4096, 32768]


@pytest.fixture(scope="module")
def env():
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _lib.set_plane_format(_lib.PLANES_F16)
  _lib.plane_overflow()
  yield torch, _lib, lib
  _lib.set_plane_format(before)


@pytest.mark.parametrize("B", BATCHES)
def test_fwd_thin_matches_general(env, B):
  torch, _lib, lib = env
  case = _fwd_case(torch, _lib, lib, B, FWD_OPS, seed=B + 3)
  partner = len(FWD_OPS) - 1
  fails = []
  for k in range(partner):
    thin = _fwd_run(torch, _lib, lib, case, [k])[0]
    general = _fwd_run(torch, _lib, lib, case, [k, partner])[0]
    fails += _fwd_check(torch, _lib, lib, case, k, thin)
    if not _bytes_equal(thin, general):
      fails.append("op %d: pl_thin_kernel and pl_gemm_kernel outputs differ" % k)
  assert not fails, "\n".join(fails)


@pytest.mark.parametrize("B", [129, 4096])
def test_fwd_thin_dropout_row0(env, B):
  """a row slice of the minibatch (dropout_row0 != 0) draws the same mask on both kernels"""
  torch, _lib, lib = env
  case = _fwd_case(torch, _lib, lib, B, [FWD_OPS[4], FWD_OPS[-1]], seed=B + 5)
  outs = []
  for idx in ([0], [0, 1]):
    bufs = [torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, case["ops"][i]["O"]) // 4,), device="cuda") for i in idx]
    structs = [_fwd_struct(_lib, case, case["ops"][i], buf) for i, buf in zip(idx, bufs)]
    for s in structs:
      s.dropout_row0 = 1000
    _lib.check(lib.adn_dense_fwd_p_group((_lib.FwdOp * len(structs))(*structs), len(structs), B, _stream(torch)),
               "adn_dense_fwd_p_group")
    outs.append(bufs[0])
  assert _bytes_equal(outs[0], outs[1])


def _colsum_part(f, B, I, O):
  """the per-32-row column sums the dX epilogue wrote into the op's workspace (dense_bwd_workspace_bytes layout)"""
  import torch
  max_s = min(64, max(1, (16 << 20) // max(1, I * O)))
  base = (f["ws"].data_ptr() + 255) // 256 * 256 - f["ws"].data_ptr()
  off = base + (max_s * I * O * 4 + 255) // 256 * 256
  rows = (B + 31) // 32
  return f["ws"][off:off + rows * I * 4].view(torch.float32).reshape(rows, I)


@pytest.mark.parametrize("B", BATCHES)
def test_dx_thin_matches_general(env, B):
  torch, _lib, lib = env
  case = _bwd_case(torch, _lib, lib, B, BWD_OPS, seed=B + 11)
  partner = len(BWD_OPS) - 1
  fails = []
  for k in range(partner):
    d = case["ops"][k]
    thin = _bwd_run(torch, _lib, lib, case, [k])[0]
    general = _bwd_run(torch, _lib, lib, case, [k, partner])[0]
    fails += _bwd_check(torch, _lib, lib, case, k, thin)
    for key in ("dxp", "cs"):
      if thin[key] is not None and not _bytes_equal(thin[key], general[key]):
        fails.append("op %d: %s differs between pl_thin_kernel and pl_gemm_kernel" % (k, key))
    if thin["cs"] is not None and not _bytes_equal(_colsum_part(thin, B, d["I"], d["O"]),
                                                   _colsum_part(general, B, d["I"], d["O"])):
      fails.append("op %d: per-32-row column sums differ between the kernels" % k)
  assert not _lib.plane_overflow()
  assert not fails, "\n".join(fails)


def test_kernel_choice(env):
  torch, _lib, lib = env
  B = 256
  case = _fwd_case(torch, _lib, lib, B, FWD_OPS, seed=1)
  thin = _kernels(torch, lambda: _fwd_run(torch, _lib, lib, case, list(range(8))))
  assert len(thin) == 1 and "pl_thin_kernel" in thin[0], thin
  mixed = _kernels(torch, lambda: _fwd_run(torch, _lib, lib, case, [0, 8]))
  assert len(mixed) == 1 and "pl_gemm_kernel" in mixed[0], mixed
  nine = _kernels(torch, lambda: _fwd_run(torch, _lib, lib, case, list(range(8)) + [0]))
  assert len(nine) == 2 and all("pl_thin_kernel" in n for n in nine), nine
  bcase = _bwd_case(torch, _lib, lib, B, BWD_OPS, seed=2)
  dx = _kernels(torch, lambda: _bwd_run(torch, _lib, lib, bcase, list(range(6))))
  assert len(dx) == 1 and "pl_thin_kernel" in dx[0], dx
  try:
    _lib.set_plane_format(_lib.PLANES_TF32)
    tcase = _fwd_case(torch, _lib, lib, B, FWD_OPS[:2], seed=3)
    tf32 = _kernels(torch, lambda: _fwd_run(torch, _lib, lib, tcase, [0, 1]))
  finally:
    _lib.set_plane_format(_lib.PLANES_F16)
  assert len(tf32) == 1 and "pl_gemm_kernel" in tf32[0], tf32
