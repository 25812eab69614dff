"""The wide forward / dX plane GEMM (csrc/planes.cu pl_wide_kernel): single-source fp16 forward and dX groups with
planes out, that are not thin-K groups, whose MMA work grows by at most 1/8 when every N is padded to 128 columns and
whose wide work items still spread over the SMs, run on 128 x 128 tiles; the others keep their kernels.

Each op runs on the wide kernel -- alone at B = 32768; at smaller batches a group of one op has too few work items for
128 x 128 tiles, so there the ops run as one group -- and again in one call beside a partner with a dense fp32 output
(the group then takes pl_gemm_kernel); the two results must agree byte for byte -- hi and lo' planes, sign-bit words, the per-32-row column
sums and their reduction -- and each is checked against float64 with the componentwise bounds of
test_gpu_plane_groups.  N is not a multiple of 128 in most ops, so the second 64-column unit of the last tile lies
partly or wholly past the output.

The kernel-choice checks read kernel names from torch.profiler in a child process (tests/plane_kernels.py).
"""

import pytest

from tests.plane_kernels import in_child, kernels as _kernels
from tests.test_gpu_plane_groups import (DX_MUL, _bwd_case, _bwd_check, _bwd_run, _bytes_equal, _fwd_case, _fwd_check,
                                         _fwd_run, _fwd_struct, _open, _stream)
from tests.test_gpu_thin_k import _colsum_part

pytestmark = pytest.mark.gpu

# forward ops (in, out, bias, act, planes out, dropout): K in 129..1024, N in {200, 450, 1000, 1024}
FWD_OPS = [
    (129, 200, 1, 1, 1, None),
    (256, 1000, 0, 0, 1, None),
    (300, 450, 1, 1, 1, (5, 0)),
    (777, 200, 1, 0, 1, (6, 1)),
    (1024, 1024, 1, 1, 1, (7, 2)),
    (777, 1000, 0, 1, 1, (8, 3)),
    (129, 1024, 1, 0, 1, None),
    (640, 1000, 1, 1, 1, None),
]
FWD_PARTNER = (64, 10, 1, 0, 0, None)         # dense fp32 output: the group runs on pl_gemm_kernel
# backward ops (in, out, x_relu_mask, dz_log2_scale, dx_mul, outputs): dX has N = in, K = out
BWD_OPS = [
    (200, 129, 1, 7, 0.0, "dxp cs"),
    (1000, 256, 0, 0, DX_MUL, "dxp cs"),
    (450, 300, 1, 15, DX_MUL, "dxp"),
    (200, 777, 0, 7, 0.0, "dxp"),
    (1024, 1024, 1, 15, 0.0, "dxp cs"),
    (1000, 777, 1, 0, 0.0, "dxp cs"),
    (1024, 129, 0, 7, DX_MUL, "dxp"),
    (1000, 640, 1, 15, 0.0, "dxp cs"),
]
BWD_PARTNER = (64, 10, 0, 0, 0.0, "dx")       # dense fp32 dX: the group runs on pl_gemm_kernel
# per batch: the calls that run the ops on pl_wide_kernel (lists of op indices; test_kernel_choice confirms the kernel)
WIDE_CALLS = {1500: [list(range(8))], 4097: [[0, 1, 2, 3, 4]], 32768: [[k] for k in range(5)]}
BATCHES = sorted(WIDE_CALLS)


@pytest.fixture(scope="module")
def env():
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _lib.set_plane_format(_lib.PLANES_F16)
  _lib.plane_overflow()
  yield torch, _lib, lib
  _lib.set_plane_format(before)


def _ops(B, ops):
  """the ops of the batch's wide calls, renumbered, and the calls"""
  used = sorted({k for call in WIDE_CALLS[B] for k in call})
  return [ops[k] for k in used], [[used.index(k) for k in call] for call in WIDE_CALLS[B]]


@pytest.mark.parametrize("B", BATCHES)
def test_fwd_wide_matches_general(env, B):
  torch, _lib, lib = env
  fwd, calls = _ops(B, FWD_OPS)
  case = _fwd_case(torch, _lib, lib, B, fwd + [FWD_PARTNER], seed=B + 41)
  partner = len(fwd)
  fails = []
  for call in calls:
    for k, wide in zip(call, _fwd_run(torch, _lib, lib, case, call)):
      general = _fwd_run(torch, _lib, lib, case, [k, partner])[0]
      fails += _fwd_check(torch, _lib, lib, case, k, wide)
      if not _bytes_equal(wide, general):
        fails.append("op %d: pl_wide_kernel and pl_gemm_kernel outputs differ" % k)
  assert not _lib.plane_overflow()
  assert not fails, "\n".join(fails)


@pytest.mark.parametrize("B", [4096, 32768])
def test_fwd_wide_dropout_row0(env, B):
  """a row slice of the minibatch (dropout_row0 != 0) draws the same mask on both kernels"""
  torch, _lib, lib = env
  case = _fwd_case(torch, _lib, lib, B, [FWD_OPS[2], FWD_PARTNER], seed=B + 43)
  outs = []
  for idx in ([0], [0, 1]):
    bufs = [torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, case["ops"][i]["O"]) // 4,), device="cuda")
            if case["ops"][i]["planes"] else torch.zeros((B, case["ops"][i]["O"]), device="cuda") for i in idx]
    structs = [_fwd_struct(_lib, case, case["ops"][i], buf) for i, buf in zip(idx, bufs)]
    for s in structs:
      s.dropout_row0 = 1000
    _lib.check(lib.adn_dense_fwd_p_group((_lib.FwdOp * len(structs))(*structs), len(structs), B, _stream(torch)),
               "adn_dense_fwd_p_group")
    outs.append(bufs[0])
  assert _bytes_equal(outs[0], outs[1])


@pytest.mark.parametrize("B", BATCHES)
def test_dx_wide_matches_general(env, B):
  torch, _lib, lib = env
  bwd, calls = _ops(B, BWD_OPS)
  case = _bwd_case(torch, _lib, lib, B, bwd + [BWD_PARTNER], seed=B + 47)
  partner = len(bwd)
  fails = []
  for call in calls:
    for k, wide in zip(call, _bwd_run(torch, _lib, lib, case, call)):
      d = case["ops"][k]
      general = _bwd_run(torch, _lib, lib, case, [k, partner])[0]
      fails += _bwd_check(torch, _lib, lib, case, k, wide)
      for key in ("dxp", "cs"):
        if wide[key] is not None and not _bytes_equal(wide[key], general[key]):
          fails.append("op %d: %s differs between pl_wide_kernel and pl_gemm_kernel" % (k, key))
      if wide["cs"] is not None and not _bytes_equal(_colsum_part(wide, B, d["I"], d["O"]),
                                                     _colsum_part(general, B, d["I"], d["O"])):
        fails.append("op %d: per-32-row column sums differ between the kernels" % k)
  assert not _lib.plane_overflow()
  assert not fails, "\n".join(fails)


def _choice_groups():
  """kernel names of single forward / dX group calls: [(label, names)]"""
  torch, _lib, lib = _open()
  _lib.set_plane_format(_lib.PLANES_F16)
  out = []
  B = 256
  fcase = _fwd_case(torch, _lib, lib, B, FWD_OPS[:4] + [FWD_PARTNER, (256, 320, 1, 1, 1, None), (100, 200, 1, 1, 1, None)],
                    seed=1)
  for label, idx in (("fwd few items", [0, 1, 2, 3]), ("fwd+dense", [1, 4]), ("fwd 320", [5]), ("fwd thin", [6])):
    out.append((label, _kernels(torch, lambda: _fwd_run(torch, _lib, lib, fcase, idx))))
  # N = 576: 9 narrow tiles, 5 wide ones (+11 % MMA work); with 128-row blocks = SMs // 5 + 1 the 5 wide tiles of
  # every block take two rounds of the SMs, as many as the 9 narrow ones
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  Bi = 128 * (sms // 5 + 1)
  icase = _fwd_case(torch, _lib, lib, Bi, [(256, 576, 1, 1, 1, None)], seed=2)
  out.append(("fwd imbalance", _kernels(torch, lambda: _fwd_run(torch, _lib, lib, icase, [0]))))
  bcase = _bwd_case(torch, _lib, lib, B, BWD_OPS[:4] + [BWD_PARTNER, (64, 100, 1, 0, 0.0, "dxp cs")], seed=3)
  for label, idx in (("dx few items", [0, 1, 2, 3]), ("dx+dense", [1, 4]), ("dx thin", [5])):
    out.append((label, _kernels(torch, lambda: _bwd_run(torch, _lib, lib, bcase, idx))))
  _lib.set_plane_format(_lib.PLANES_TF32)
  tcase = _fwd_case(torch, _lib, lib, B, FWD_OPS[:2], seed=4)
  out.append(("tf32", _kernels(torch, lambda: _fwd_run(torch, _lib, lib, tcase, [0, 1]))))
  _lib.set_plane_format(_lib.PLANES_F16)
  for Bw in sorted(WIDE_CALLS):          # the wide calls of the byte comparisons above
    ops, calls = _ops(Bw, FWD_OPS)
    wcase = _fwd_case(torch, _lib, lib, Bw, ops, seed=5)
    for call in calls:
      out.append(("fwd B=%d %s" % (Bw, call), _kernels(torch, lambda: _fwd_run(torch, _lib, lib, wcase, call))))
    ops, calls = _ops(Bw, BWD_OPS)
    wcase = _bwd_case(torch, _lib, lib, Bw, ops, seed=6)
    for call in calls:
      out.append(("dx B=%d %s" % (Bw, call), _kernels(torch, lambda: _bwd_run(torch, _lib, lib, wcase, call))))
  return out


def test_kernel_choice(env):
  # 64 x 4 ... 13 k-blocks on 2 row blocks: too few items to fill the SMs twice over, so wide tiles would leave the
  # busiest CTA twice the work
  want = {"fwd few items": ["pl_gemm_kernel<1, 0>"],
          "fwd+dense": ["pl_gemm_kernel<1, 0>"],          # a dense fp32 output keeps the group on pl_gemm_kernel
          "fwd 320": ["pl_gemm_kernel<1, 0>"],            # padding 320 columns to 384 adds 1/5
          "fwd thin": ["pl_thin_kernel<0>"],              # K <= 128: pl_thin_kernel keeps priority
          "fwd imbalance": ["pl_gemm_kernel<1, 0>"],
          "dx few items": ["pl_gemm_kernel<1, 1>"],
          "dx+dense": ["pl_gemm_kernel<1, 1>"],
          "dx thin": ["pl_thin_kernel<1>"],
          "tf32": ["pl_gemm_kernel<0, 0>"]}
  for Bw in sorted(WIDE_CALLS):
    for kind, epi, ops in (("fwd", 0, FWD_OPS), ("dx", 1, BWD_OPS)):
      for call in _ops(Bw, ops)[1]:
        want["%s B=%d %s" % (kind, Bw, call)] = ["pl_wide_kernel<%d>" % epi]
  got = in_child("test_gpu_wide_fwd", "_choice_groups")
  assert [label for label, _ in got] == list(want), got
  for label, names in got:
    assert names == want[label], (label, names)


def test_bench_step_kernel_choice(env):
  """The benchmarked training step (bench.py's 8 candidates 100 -> H -> H -> 10): its hidden-layer forward and dX
  launches run pl_wide_kernel; the first-layer forward (K = 100) and the logits layer's dX (K = 10) stay on
  pl_thin_kernel, and no dX runs on pl_gemm_kernel."""
  seq = in_child("plane_kernels", "bench_step_kernels")
  for k in ("pl_wide_kernel<0>", "pl_wide_kernel<1>", "pl_thin_kernel<0>", "pl_thin_kernel<1>"):
    assert seq.count(k) == 1, seq
  assert "pl_gemm_kernel<1, 1>" not in seq, seq
  # forward: first layer, then the hidden layer; backward: the logits layer's dX, then the hidden layer's
  assert (seq.index("pl_thin_kernel<0>") < seq.index("pl_wide_kernel<0>") < seq.index("pl_thin_kernel<1>") <
          seq.index("pl_wide_kernel<1>")), seq
