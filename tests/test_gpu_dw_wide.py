"""The wide dW plane GEMM (csrc/planes.cu pl_dw_kernel): fp16 dW groups whose MMA work grows by at most 1/8 when every
N is padded to 128 columns instead of 64, and whose wide work items still spread over the SMs, run on 128 x 128 tiles;
every other dW group runs on pl_gemm_kernel.

Each dW op runs in one call beside a 20 x 2048 op (the group runs on pl_dw_kernel) and again beside a 4096 x 10 op
(N = 10: the group runs on pl_gemm_kernel).  The split-K plan is chosen for the whole group, from the work-item count,
the split cap and the partial-sum bytes of every op; the two companions have the same 32 tiles of 128 x 64, the same
cap of 64 splits and the same 40,960 entries, so both calls run the op on the same split plan.  The test reads the
number of partial sums each call wrote back from the op's workspace to show that, then requires dW to agree byte for
byte.  Every result is also checked against float64 with the componentwise bounds of test_gpu_plane_groups.

The kernel-choice checks read kernel names from torch.profiler in a child process (tests/plane_kernels.py).
"""

import pytest

from tests.plane_kernels import in_child, kernels as _kernels
from tests.test_gpu_plane_groups import _bwd_bufs, _bwd_call, _bwd_case, _bwd_check, _bwd_struct, _bytes_equal, _open

pytestmark = pytest.mark.gpu

# dW-only ops (in, out, x_relu_mask, dz_log2_scale, dx_mul, outputs): in in {1, 33, 100, 128, 200, 1024}, out in
# {64, 65, 128, 200, 1024}, scales 2^0 / 2^7 / 2^15
OPS = [
    (1, 65, 0, 0, 0.0, "dw"),
    (33, 200, 1, 7, 0.0, "dw"),
    (100, 1024, 0, 15, 0.0, "dw"),
    (128, 128, 1, 0, 0.0, "dw"),
    (200, 65, 0, 7, 0.0, "dw"),
    (1024, 1024, 1, 15, 0.0, "dw"),
    (100, 64, 0, 0, 0.0, "dw"),
    (1024, 200, 0, 7, 0.0, "dw"),
    (200, 1024, 1, 15, 0.0, "dw"),
    (128, 64, 0, 7, 0.0, "dw"),
]
WIDE = (20, 2048, 0, 0, 0.0, "dw")        # 1 x 32 tiles of 128 x 64, split cap 64: the group stays wide
NARROW = (4096, 10, 0, 7, 0.0, "dw")      # 32 x 1 tiles, split cap 64, N = 10: the group goes to pl_gemm_kernel
BATCHES = [1, 129, 4096, 32768]


@pytest.fixture(scope="module")
def env():
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _lib.set_plane_format(_lib.PLANES_F16)
  _lib.plane_overflow()
  yield torch, _lib, lib
  _lib.set_plane_format(before)


def _run(torch, _lib, lib, case, idx):
  """dW of ops idx in one call; workspaces filled with NaN words first, so that the split-K partials written can be
  counted afterwards"""
  B = case["B"]
  bufs = [_bwd_bufs(torch, _lib, B, case["ops"][i]) for i in idx]
  for f in bufs:
    f["ws"].fill_(0xFF)
  structs = [_bwd_struct(_lib, case["ops"][i], f) for i, f in zip(idx, bufs)]
  _lib.check(_bwd_call(torch, _lib, lib, B, structs), "adn_dense_bwd_p_group")
  return bufs


def _splits(torch, f, I, O):
  """split-K partial sums the call wrote into the op's workspace (dense_bwd_workspace_bytes layout); 1 = dW written
  directly.  A split size is ceil(k-blocks / s) for a split count s, so equal counts mean equal split boundaries."""
  max_s = min(64, max(1, (16 << 20) // max(1, I * O)))
  base = (f["ws"].data_ptr() + 255) // 256 * 256 - f["ws"].data_ptr()
  part = f["ws"][base:base + max_s * I * O * 4].view(torch.int32).reshape(max_s, I * O)
  return max(1, int((part[:, 0] != -1).sum().item()))


@pytest.mark.parametrize("B", BATCHES)
def test_dw_wide_matches_general(env, B):
  torch, _lib, lib = env
  case = _bwd_case(torch, _lib, lib, B, OPS + [WIDE, NARROW], seed=B + 29)
  wide_c, narrow_c = len(OPS), len(OPS) + 1
  fails, split_counts = [], set()
  for k, (I, O) in enumerate((o[0], o[1]) for o in OPS):
    wide = _run(torch, _lib, lib, case, [k, wide_c])
    general = _run(torch, _lib, lib, case, [k, narrow_c])
    fails += _bwd_check(torch, _lib, lib, case, k, wide[0])
    fails += _bwd_check(torch, _lib, lib, case, k, general[0])
    if k == 0:
      fails += _bwd_check(torch, _lib, lib, case, wide_c, wide[1])
      fails += _bwd_check(torch, _lib, lib, case, narrow_c, general[1])
    s_wide, s_general = _splits(torch, wide[0], I, O), _splits(torch, general[0], I, O)
    split_counts.add(s_wide)
    if s_wide != s_general:
      fails.append("op %d (%d x %d): %d splits beside the wide companion, %d beside the narrow one" %
                   (k, I, O, s_wide, s_general))
    elif not _bytes_equal(wide[0]["dw"], general[0]["dw"]):
      fails.append("op %d (%d x %d, %d splits): dW differs between pl_dw_kernel and pl_gemm_kernel" % (k, I, O, s_wide))
  assert not _lib.plane_overflow()
  assert not fails, "\n".join(fails)
  if B >= 4096:      # the byte comparisons above include split-K plans, not only the direct epilogue
    assert max(split_counts) > 1, split_counts


def _choice_groups():
  """kernel names of single dW group calls, fp16 and TF32: [(label, names)]"""
  torch, _lib, lib = _open()
  _lib.set_plane_format(_lib.PLANES_F16)
  B = 256
  case = _bwd_case(torch, _lib, lib, B, OPS + [WIDE, NARROW], seed=1)
  wide_c, narrow_c = len(OPS), len(OPS) + 1
  out = []
  for label, idx in (("200x65", [4]), ("100x64", [6]), ("100x64+wide", [6, wide_c]), ("100x64+narrow", [6, narrow_c]),
                     ("1024x1024+narrow", [5, narrow_c])):
    out.append((label, _kernels(torch, lambda: _run(torch, _lib, lib, case, idx))))
  _lib.set_plane_format(_lib.PLANES_TF32)
  tcase = _bwd_case(torch, _lib, lib, B, OPS[:3], seed=3)
  out.append(("tf32", _kernels(torch, lambda: _run(torch, _lib, lib, tcase, [0, 1, 2]))))
  return out


def test_kernel_choice(env):
  want = {"200x65": "pl_dw_kernel",                 # padding 65 columns to 128 costs nothing
          "100x64": "pl_gemm_kernel<1, 2>",         # padding 64 columns to 128 doubles the work
          "100x64+wide": "pl_dw_kernel",
          "100x64+narrow": "pl_gemm_kernel<1, 2>",
          "1024x1024+narrow": "pl_gemm_kernel<1, 2>",
          "tf32": "pl_gemm_kernel<0, 2>"}
  got = in_child("test_gpu_dw_wide", "_choice_groups")
  assert [label for label, _ in got] == list(want), got
  for label, names in got:
    assert len(names) == 1 and want[label] in names[0], (label, names)


def test_bench_step_kernel_choice(env):
  """The benchmarked training step (bench.py's 8 candidates 100 -> H -> H -> 10): its hidden-layer dW launch runs
  pl_dw_kernel.  The logits-layer dW (N = 10) runs pl_gemm_kernel<fp16, EPI_PARTIAL>, and so does the first-layer dW,
  whose 135 wide work items would leave three SMs with two each."""
  names = in_child("plane_kernels", "bench_step_kernels")
  dw = [n for n in names if "pl_dw_kernel" in n or "pl_gemm_kernel<1, 2>" in n]
  # the backward visits the logits layer first, then the hidden layer, then the first layer
  assert len(dw) == 3, names
  assert "pl_gemm_kernel<1, 2>" in dw[0] and "pl_dw_kernel" in dw[1] and "pl_gemm_kernel<1, 2>" in dw[2], dw
