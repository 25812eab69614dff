"""GPU parity of the plane-native tensor-core pipeline (csrc/planes.cu) through the C ABI, in BOTH plane formats
(fp16 hi/lo' planes with fp16 MMAs -- the default -- and the TF32 fallback, csrc/plane_fmt.cuh).

Checked against fp64 NumPy restatements of the reference arithmetic
(tf.layers.dense and its gradients, adanet/examples/simple_dnn.py:72-86,103-110)
with the forward-error bound of an fp32 GEMM: |err| <= 3e-6 * max(|A| @ |B|)
(the same bound tests/test_gpu_kernels.py uses for the fp32 ABI).
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL = 3e-6


@pytest.fixture(scope="module", params=["f16", "tf32"])
def env(request):
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  before = _lib.plane_format()
  _lib.set_plane_format(_lib.PLANES_F16 if request.param == "f16" else _lib.PLANES_TF32)
  _lib.plane_overflow()      # clear the sticky flag
  yield torch, _lib, lib
  _lib.set_plane_format(before)


def _layout(_lib, pl, r, c):
  """(hi plane as float64 [nkb, r, BK], sign-bit words [nb32, r]) of a plane tensor in the current format"""
  f16 = _lib.plane_format() == _lib.PLANES_F16
  bk = 64 if f16 else 32
  nkb = (c + bk - 1) // bk
  elems = -(-(nkb * r * bk) // 128) * 128
  raw = pl.cpu().numpy()
  if f16:
    hi = raw.view(np.float16)[: nkb * r * bk].reshape(nkb, r, bk)
    off_words = 2 * elems * 2 // 4
  else:
    hi = raw[: nkb * r * bk].reshape(nkb, r, bk)
    off_words = 2 * elems
  nb32 = nkb * (bk // 32)
  bits = raw[off_words: off_words + nb32 * r].view(np.uint32).reshape(nb32, r)
  return hi, bits, bk


def _planes(torch, _lib, lib, a, log2_scale=0):
  """dense numpy [r,c] (times 2^log2_scale) -> zero-initialised plane tensor on the GPU"""
  r, c = a.shape
  nb = _lib.query(_lib.Q_PLANES_BYTES, r, c)
  pl = torch.zeros((nb // 4,), dtype=torch.float32, device="cuda")
  src = torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).cuda()
  _lib.check(lib.adn_planes_split_scaled(src.data_ptr(), r, c, pl.data_ptr(), log2_scale,
                                         torch.cuda.current_stream().cuda_stream), "split")
  return pl


def _merge(torch, _lib, lib, pl, r, c):
  out = torch.empty((r, c), dtype=torch.float32, device="cuda")
  _lib.check(lib.adn_planes_merge(pl.data_ptr(), r, c, out.data_ptr(), torch.cuda.current_stream().cuda_stream), "merge")
  return out.cpu().numpy()


def _relerr(got, exact, scale=None):
  """max |err| relative to `scale` (default: max |exact|)"""
  if scale is None:
    scale = np.abs(exact).max() + 1e-30
  return float(np.abs(got.astype(np.float64) - exact).max() / scale)


def _bound(a, b):
  return float((np.abs(a).astype(np.float64) @ np.abs(b).astype(np.float64)).max())


@pytest.mark.parametrize("r,c", [(1, 1), (37, 100), (128, 32), (300, 130), (4096, 1024)])
def test_split_merge_roundtrip(env, r, c):
  torch, _lib, lib = env
  rng = np.random.default_rng(r * 1000 + c)
  a = rng.standard_normal((r, c)).astype(np.float32)
  pl = _planes(torch, _lib, lib, a)
  back = _merge(torch, _lib, lib, pl, r, c)
  assert np.abs(back - a).max() <= 2.0 ** -22 * np.abs(a).max()
  # padding columns of the last k-block are exact zeros, hi carries 11 significant bits
  hi, bits, bk = _layout(_lib, pl, r, c)
  if c % bk:
    assert (hi[-1, :, c % bk:] == 0).all()
  if hi.dtype == np.float32:
    assert (hi.view(np.uint32) & 0x1FFF == 0).all()
  # sign bits [cols/32][rows]: bit j of word (q, row) <=> a[row, q*32+j] > 0
  nb32 = bits.shape[0]
  pad = np.zeros((r, nb32 * 32), dtype=bool)
  pad[:, :c] = a > 0
  want_bits = (pad.reshape(r, nb32, 32) * (np.uint64(1) << np.arange(32, dtype=np.uint64))).sum(axis=2).astype(np.uint32).T
  assert np.array_equal(bits, want_bits)


SHAPES = [(128, 32, 64), (300, 100, 70), (512, 1024, 256), (1000, 257, 10), (2048, 64, 1024), (129, 33, 129)]


@pytest.mark.parametrize("B,I,O", SHAPES)
@pytest.mark.parametrize("act", [0, 1])
def test_dense_fwd_planes(env, B, I, O, act):
  torch, _lib, lib = env
  rng = np.random.default_rng(B + I + O)
  x = rng.standard_normal((B, I)).astype(np.float32)
  w = (rng.standard_normal((I, O)) / np.sqrt(I)).astype(np.float32)
  b = rng.standard_normal((O,)).astype(np.float32)
  exact = x.astype(np.float64) @ w.astype(np.float64) + b
  if act:
    exact = np.maximum(exact, 0)
  xp, wp = _planes(torch, _lib, lib, x), _planes(torch, _lib, lib, w)
  bd = torch.as_tensor(b).cuda()
  sp = torch.cuda.current_stream().cuda_stream
  # dense fp32 output
  y = torch.full((B, O), float("nan"), device="cuda")
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), bd.data_ptr(), None, y.data_ptr(), B, I, O, act, sp), "fwd_p")
  sc = _bound(x, w) + np.abs(b).max()
  assert _relerr(y.cpu().numpy(), exact, sc) < TOL
  # plane output (what the next layer consumes)
  yp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, O) // 4,), device="cuda")
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), bd.data_ptr(), yp.data_ptr(), None, B, I, O, act, sp), "fwd_p")
  assert _relerr(_merge(torch, _lib, lib, yp, B, O), exact, sc) < TOL
  hi, bits, bk = _layout(_lib, yp, B, O)
  if O % bk:
    assert (hi[-1, :, O % bk:] == 0).all()
  # sign bits written by the epilogue agree with the stored values
  pos = (hi > 0).transpose(1, 0, 2).reshape(B, -1, 32)               # [B, nb32, 32]
  want_bits = (pos * (np.uint64(1) << np.arange(32, dtype=np.uint64))).sum(axis=2).astype(np.uint32).T
  assert np.array_equal(bits, want_bits)


@pytest.mark.parametrize("B,I,O", SHAPES)
@pytest.mark.parametrize("mask", [0, 1])
def test_dense_bwd_planes(env, B, I, O, mask):
  torch, _lib, lib = env
  rng = np.random.default_rng(7 * B + I + O)
  x = rng.standard_normal((B, I)).astype(np.float32)
  if mask:
    x = np.maximum(x, 0)          # a ReLU output: the mask is x > 0
  w = (rng.standard_normal((I, O)) / np.sqrt(O)).astype(np.float32)
  dz = rng.standard_normal((B, O)).astype(np.float32)
  dw_exact = x.astype(np.float64).T @ dz.astype(np.float64)
  dx_exact = dz.astype(np.float64) @ w.astype(np.float64).T
  if mask:
    dx_exact = dx_exact * (x > 0)
  cs_exact = dx_exact.sum(axis=0)
  xp, wp, dzp = (_planes(torch, _lib, lib, a) for a in (x, w, dz))
  nb = _lib.query(_lib.Q_DENSE_BWD_P_WS, B, I, O)
  ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")
  sp = torch.cuda.current_stream().cuda_stream
  dw = torch.full((I, O), float("nan"), device="cuda")
  dxp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, I) // 4,), device="cuda")
  cs = torch.full((I,), float("nan"), device="cuda")
  _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), wp.data_ptr(), dzp.data_ptr(), dxp.data_ptr(), None, cs.data_ptr(),
                                 dw.data_ptr(), B, I, O, mask, 0, ws.data_ptr(), nb, sp), "bwd_p")
  s_dw, s_dx = _bound(x.T, dz), _bound(dz, w.T)
  assert _relerr(dw.cpu().numpy(), dw_exact, s_dw) < TOL
  assert _relerr(_merge(torch, _lib, lib, dxp, B, I), dx_exact, s_dx) < TOL
  assert _relerr(cs.cpu().numpy(), cs_exact, np.abs(dx_exact).sum(axis=0).max()) < TOL
  # dense dx variant, no dw
  dx = torch.full((B, I), float("nan"), device="cuda")
  _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), wp.data_ptr(), dzp.data_ptr(), None, dx.data_ptr(), None, None, B, I, O,
                                 mask, 0, ws.data_ptr(), nb, sp), "bwd_p")
  assert _relerr(dx.cpu().numpy(), dx_exact, s_dx) < TOL


def test_large_batch_dw_split_k(env):
  """K = batch = 32768 (BASELINE configs[2] batch): split-K dW and the two-level column sums."""
  torch, _lib, lib = env
  B, I, O = 32768, 100, 192
  rng = np.random.default_rng(3)
  x = np.maximum(rng.standard_normal((B, I)), 0).astype(np.float32)
  w = (rng.standard_normal((I, O)) / np.sqrt(O)).astype(np.float32)
  dz = (rng.standard_normal((B, O)) / B).astype(np.float32)
  # the gradient (O(1/B): below fp16's normal range) travels as dz * 2^15; dW / db come back un-scaled, dX planes
  # keep the scale
  LOG2 = 15
  xp, wp = (_planes(torch, _lib, lib, a) for a in (x, w))
  dzp = _planes(torch, _lib, lib, dz, LOG2)
  nb = _lib.query(_lib.Q_DENSE_BWD_P_WS, B, I, O)
  ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")
  dw = torch.empty((I, O), device="cuda")
  cs = torch.empty((I,), device="cuda")
  dxp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, I) // 4,), device="cuda")
  _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), wp.data_ptr(), dzp.data_ptr(), dxp.data_ptr(), None, cs.data_ptr(),
                                 dw.data_ptr(), B, I, O, 1, LOG2, ws.data_ptr(), nb, torch.cuda.current_stream().cuda_stream),
             "bwd_p")
  assert _relerr(dw.cpu().numpy(), x.astype(np.float64).T @ dz.astype(np.float64), _bound(x.T, dz)) < TOL
  dx_exact = (dz.astype(np.float64) @ w.astype(np.float64).T) * (x > 0)
  assert _relerr(cs.cpu().numpy(), dx_exact.sum(axis=0), np.abs(dx_exact).sum(axis=0).max()) < TOL
  assert _relerr(_merge(torch, _lib, lib, dxp, B, I) / 2.0 ** LOG2, dx_exact, _bound(dz, w.T)) < TOL
  assert not _lib.plane_overflow()


def test_opt_step_planes(env):
  torch, _lib, lib = env
  rng = np.random.default_rng(5)
  sp = torch.cuda.current_stream().cuda_stream
  # SGD step that refreshes the planes of a [100, 70] kernel; bias has no planes
  w = rng.standard_normal((100, 70)).astype(np.float32)
  g = rng.standard_normal((100, 70)).astype(np.float32)
  b, gb = rng.standard_normal((70,)).astype(np.float32), rng.standard_normal((70,)).astype(np.float32)
  wd, gd, bd, gbd = (torch.as_tensor(t).cuda() for t in (w, g, b, gb))
  wp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, 100, 70) // 4,), device="cuda")
  _lib.check(lib.adn_opt_step_p(_lib.OPT_SGD, _lib.ptr_array([wd.data_ptr(), bd.data_ptr()]),
                                _lib.ptr_array([gd.data_ptr(), gbd.data_ptr()]), None, None, _lib.i64_array([7000, 70]), 2,
                                _lib.f32_array([0.1]), None, _lib.ptr_array([wp.data_ptr(), None]), _lib.i64_array([70, 0]),
                                sp), "opt_step_p")
  want = (w - np.float32(0.1) * g).astype(np.float32)
  assert np.array_equal(wd.cpu().numpy(), want)
  assert np.array_equal(bd.cpu().numpy(), (b - np.float32(0.1) * gb).astype(np.float32))
  ref = _planes(torch, _lib, lib, want)
  f16 = _lib.plane_format() == _lib.PLANES_F16
  n2 = (2 * 100 * 128 * 2 // 4) if f16 else (2 * 100 * 96)    # hi + lo planes of a [100, 70] tensor in float32 words
  assert torch.equal(wp[:n2], ref[:n2])


def test_fp16_overflow_flag(env):
  """A finite value that does not fit fp16 raises the sticky flag (and only in the fp16 format): what makes the
  search fall back to TF32 planes for the iteration."""
  torch, _lib, lib = env
  a = np.ones((64, 40), dtype=np.float32)
  _planes(torch, _lib, lib, a)
  assert not _lib.plane_overflow()
  a[3, 7] = 70000.0
  _planes(torch, _lib, lib, a)
  assert _lib.plane_overflow() == (_lib.plane_format() == _lib.PLANES_F16)
  assert not _lib.plane_overflow()       # reading clears it
  a[3, 7] = np.inf                       # a diverged value is not an overflow of the format
  _planes(torch, _lib, lib, a)
  assert not _lib.plane_overflow()
  # a GEMM result beyond the range (300 * 300 = 90000 in one output element) is not tracked element by element in the
  # epilogue (it would cost two instructions per value on an issue-bound path): it becomes Inf in the fp16 planes,
  # turns the losses that depend on it non-finite, and AdaNetSearch.restart_on_tf32_if_overflowed treats a non-finite
  # candidate loss under fp16 planes like the flag
  x = np.zeros((128, 64), dtype=np.float32); x[5, 0] = 300.0
  w = np.zeros((64, 64), dtype=np.float32); w[0, 9] = 300.0
  xp, wp = _planes(torch, _lib, lib, x), _planes(torch, _lib, lib, w)
  yp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, 128, 64) // 4,), device="cuda")
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, yp.data_ptr(), None, 128, 64, 64, 0,
                                 torch.cuda.current_stream().cuda_stream), "fwd_p")
  got = _merge(torch, _lib, lib, yp, 128, 64)
  if _lib.plane_format() == _lib.PLANES_F16:
    assert not np.isfinite(got[5, 9])
  else:
    assert got[5, 9] == 90000.0


def test_tma_descriptor_cache(env):
  """Descriptors are encoded once per (plane, shape, majorness, format) and reused by later launches."""
  torch, _lib, lib = env
  rng = np.random.default_rng(1)
  x = rng.standard_normal((256, 96)).astype(np.float32)
  w = rng.standard_normal((96, 80)).astype(np.float32)
  xp, wp = _planes(torch, _lib, lib, x), _planes(torch, _lib, lib, w)
  y = torch.empty((256, 80), device="cuda")
  sp = torch.cuda.current_stream().cuda_stream
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, None, y.data_ptr(), 256, 96, 80, 0, sp), "fwd_p")
  m0, h0 = _lib.query(_lib.Q_TMA_MAP_CACHE_MISSES), _lib.query(_lib.Q_TMA_MAP_CACHE_HITS)
  for _ in range(3):
    _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, None, y.data_ptr(), 256, 96, 80, 0, sp), "fwd_p")
  assert _lib.query(_lib.Q_TMA_MAP_CACHE_MISSES) == m0
  assert _lib.query(_lib.Q_TMA_MAP_CACHE_HITS) == h0 + 12




@pytest.mark.parametrize("B,I,O", [(300, 100, 70), (512, 64, 256), (129, 33, 129)])
def test_dense_fwd_dropout(env, B, I, O):
  """tf.layers.dropout fused into the forward epilogue (adanet/examples/simple_dnn.py:80-81): kept values times
  1/(1-rate), dropped ones exactly zero, sign bits follow; the keep mask is the hash the oracle restates."""
  torch, _lib, lib = env
  from tests.parity_util import orc
  rng = np.random.default_rng(B + I)
  x = rng.standard_normal((B, I)).astype(np.float32)
  w = (rng.standard_normal((I, O)) / np.sqrt(I)).astype(np.float32)
  b = rng.standard_normal((O,)).astype(np.float32)
  rate, seed, layer = 0.3, 12345, 2
  xp, wp = _planes(torch, _lib, lib, x), _planes(torch, _lib, lib, w)
  bd = torch.as_tensor(b).cuda()
  sp = torch.cuda.current_stream().cuda_stream
  for step in (0, 5):
    step_dev = torch.full((), step, dtype=torch.int64, device="cuda")
    yp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, O) // 4,), device="cuda")
    op = _lib.FwdOp(xp.data_ptr(), wp.data_ptr(), bd.data_ptr(), yp.data_ptr(), None, I, O, 1, 0)
    op.dropout_rate, op.dropout_seed, op.dropout_layer, op.dropout_step_dev = rate, seed, layer, step_dev.data_ptr()
    _lib.check(lib.adn_dense_fwd_p_group((_lib.FwdOp * 1)(op), 1, B, sp), "fwd_p_group")
    got = _merge(torch, _lib, lib, yp, B, O)
    keep = orc.dropout_keep_mask(seed, layer, step, B, O, rate)
    relu = np.maximum(x.astype(np.float64) @ w.astype(np.float64) + b, 0)
    want = np.where(keep, relu / (1.0 - rate), 0.0)
    assert abs(keep.mean() - (1 - rate)) < 0.02
    assert (got[~keep] == 0).all()
    assert _relerr(got, want, (_bound(x, w) + np.abs(b).max()) / (1 - rate)) < TOL
    hi, bits, bk = _layout(_lib, yp, B, O)
    pos = (hi > 0).transpose(1, 0, 2).reshape(B, -1, 32)
    assert np.array_equal(bits, (pos * (np.uint64(1) << np.arange(32, dtype=np.uint64))).sum(axis=2).astype(np.uint32).T)
