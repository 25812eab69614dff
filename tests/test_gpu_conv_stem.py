"""GPU tests of the SimpleCNN stem kernels, in BOTH plane formats: the wgmma 3xTF32 forward (default, F in {16, 32}),
the exact-fp32 SIMT forward (ADN_CONV_PATH=simt, and every F = 48 / 64 shape), the SIMT backward (default, all eight
(channels, filters) instantiations, staged and image-only) and the fixed-order partial reduce.

Every output is compared element by element with a float64 NumPy restatement of the stem that keeps all four conv
values of every pooled window and the componentwise error bound of each.  The planes are decoded in NumPy from the
layout of csrc/plane_fmt.cuh.  The backward reference routes the gradient with the kernel's own arg-max and starts
from the kernel's own pooled output (masking), so errors do not compound.  Each bound is gamma(n) * sum|terms| with
n the longest rounding chain in the kernel's order (written out beside each bound).

Exact dyadic inputs make every kernel bit-exact whatever its summation order; there the planes, sign bits, arg-max
(first maximum in scan order, with many exact ties) and the backward outputs must match the exact reference byte for
byte.  Every output buffer is followed by a sentinel guard that must come back unchanged, and the K padding of the
planes and the unused sign bits must stay zero.
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F32 = np.float32
ERR_INVALID, ERR_UNSUPPORTED = -22, -95
GUARD = 4096            # sentinel bytes after every output buffer
SENTINEL = 0xA5

_WORST = {}    # check name -> largest |err| / bound seen in this module (printed at teardown, pytest -s)


def _gamma(n, u=U):
  return n * u / (1.0 - n * u)


def _check(name, got, ref, bound):
  """|got - ref| <= bound element by element (bound 0 means exact).  `name` is "<where>: <check>" or "<check>";
  the report groups by <check>."""
  got = np.asarray(got, dtype=np.float64)
  ref = np.asarray(ref, dtype=np.float64)
  bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), ref.shape)
  assert got.shape == ref.shape, name
  assert np.isfinite(got).all(), "%s: non-finite output" % name
  err = np.abs(got - ref)
  bad = err > bound
  if bad.any():
    i = np.unravel_index(np.argmax(np.where(bad, err - bound, -1.0)), ref.shape)
    raise AssertionError("%s: %d elements outside the bound; at %s got %r want %r bound %r"
                         % (name, int(bad.sum()), i, got[i], ref[i], bound[i]))
  pos = bound > 0
  if pos.any():
    key = name.split(": ", 1)[-1]
    _WORST[key] = max(_WORST.get(key, 0.0), float((err[pos] / bound[pos]).max()))


@pytest.fixture(scope="module", autouse=True)
def _report():
  yield
  if _WORST:
    print("\nlargest error / bound per check:")
    for k in sorted(_WORST):
      print("  %-24s %.3g" % (k, _WORST[k]))


@pytest.fixture(scope="module", params=["f16", "tf32"])
def env(request):
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  before = _lib.plane_format()
  f16 = request.param == "f16"
  _lib.set_plane_format(_lib.PLANES_F16 if f16 else _lib.PLANES_TF32)
  _lib.plane_overflow()      # clear the sticky flag
  yield torch, _lib, lib, f16
  _lib.set_plane_format(before)


def _sp(torch):
  return torch.cuda.current_stream().cuda_stream


def _sms(_lib):
  return _lib.query(_lib.Q_SM_COUNT)


# ------------------------------------------------------------------------------------------------------------------
# shape rules mirrored from the host code
# ------------------------------------------------------------------------------------------------------------------

def _accepted(H, W, C, F):
  """conv::check_shape (csrc/conv_stem.cu)"""
  return H >= 2 and W >= 2 and H % 2 == 0 and W % 2 == 0 and C in (1, 3) and F in (16, 32, 48, 64) and \
      (H + 2) * (W + 2) * C <= 24 * 1024


def _tc_fwd_supported(H, W, C, F):
  """convtc::supported: smem_bytes<C, F> of the wgmma forward <= 227 KiB"""
  if F not in (16, 32):
    return False
  K = 16 * C
  KB = (K + 31) // 32
  nbuf = 4 if F == 16 else 2
  smem = 1024 + 2 * KB * 4 * F * 128 + 2 * 2 * KB * 128 * 128 + nbuf * (H + 2) * (W + 2) * C * 4 + F * 4
  return smem <= 227 * 1024


def _simt_groups(C, F):
  """thread groups of the SIMT backward (adn_conv_stem_bwd)"""
  g = (384 // (C * F)) & ~1
  return min(max(g, 2), 16)


def _simt_bwd_staged(H, W, C, F):
  """does the SIMT backward stage g and the arg-max words beside the image (<= 200 KiB)?"""
  pimg4 = ((H + 2) * (W + 2) * C + 3) & ~3
  cols = (H // 2) * (W // 2) * F
  smem = (2 * (pimg4 + cols + ((cols // 16 + 3) & ~3)) + _simt_groups(C, F) * (9 * C * F + F)) * 4
  return smem <= 200 * 1024


def _largest_square(C, F, pred):
  h = 2
  while _accepted(h + 2, h + 2, C, F) and pred(h + 2, h + 2, C, F):
    h += 2
  return h


# ------------------------------------------------------------------------------------------------------------------
# plane layout (csrc/plane_fmt.cuh): hi plane, lo plane, sign bits; plane [ceil(cols/BK)][rows][BK] padded to 128
# elements; bits [ceil(cols/BK) * BK/32][rows] uint32 padded to 64 words
# ------------------------------------------------------------------------------------------------------------------

class _Layout:

  def __init__(self, f16, rows, cols):
    self.f16, self.rows, self.cols = f16, rows, cols
    self.bk, self.es = (64, 2) if f16 else (32, 4)
    self.nkb = -(-cols // self.bk)
    self.n = self.nkb * rows * self.bk                       # elements of the [nkb][rows][bk] region
    self.elems = -(-self.n // 128) * 128
    self.blocks = self.nkb * (self.bk // 32)
    self.nbits = rows * self.blocks
    self.bits_words = -(-self.nbits // 64) * 64
    self.bytes = 2 * self.elems * self.es + 4 * self.bits_words
    self.bits_off = 2 * self.elems * self.es


def _alloc(torch, nbytes, fill=0):
  """a uint8 device buffer of nbytes (filled with `fill`) followed by a GUARD-byte sentinel region"""
  t = torch.full((nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
  if fill != SENTINEL:
    t[:nbytes].fill_(fill)
  return t


def _guard_ok(name, t, nbytes):
  g = t[nbytes:].cpu().numpy()
  assert (g == SENTINEL).all(), "%s: %d guard bytes after the buffer were written" % (name, int((g != SENTINEL).sum()))


def _plane_arrays(torch, buf, L, rows=None):
  """hi, lo as [nkb, rows, bk] device tensors (optionally only the given rows), and the bits [blocks, rows] words"""
  dt = torch.float16 if L.f16 else torch.float32
  hi = buf[:L.n * L.es].view(dt).view(L.nkb, L.rows, L.bk)
  lo = buf[L.elems * L.es:L.elems * L.es + L.n * L.es].view(dt).view(L.nkb, L.rows, L.bk)
  bits = buf[L.bits_off:L.bits_off + 4 * L.nbits].view(torch.int32).view(L.blocks, L.rows)
  if rows is not None:
    idx = torch.as_tensor(rows, device="cuda")
    hi, lo, bits = hi[:, idx], lo[:, idx], bits[:, idx]
  return hi, lo, bits


def _decode(torch, buf, L, rows=None):
  """values [rows, nkb*bk] (float64, exact), sign bits [rows, blocks*32] (bool)"""
  hi, lo, bits = _plane_arrays(torch, buf, L, rows)
  hi = hi.cpu().numpy().astype(np.float64)
  lo = lo.cpu().numpy().astype(np.float64)
  v = hi + lo / 2048.0 if L.f16 else hi + lo
  r = v.shape[1]
  v = v.transpose(1, 0, 2).reshape(r, L.nkb * L.bk)
  w = bits.cpu().numpy().view(np.uint32).T                           # [rows, blocks]
  b = ((w[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(r, L.blocks * 32)
  return v, b


def _padding_ok(name, torch, buf, L):
  """K-padding columns of both planes, the 128-element tails, the unused sign bits and the bits tail are zero"""
  v, b = _decode(torch, buf, L)
  assert (v[:, L.cols:] == 0).all(), "%s: K padding of the planes was written" % name
  assert not b[:, L.cols:].any(), "%s: sign bits past the last column were set" % name
  raw = buf[:L.bytes].cpu().numpy()
  for lo_, hi_ in ((L.n * L.es, L.elems * L.es), (L.elems * L.es + L.n * L.es, 2 * L.elems * L.es),
                   (L.bits_off + 4 * L.nbits, L.bytes)):
    assert (raw[lo_:hi_] == 0).all(), "%s: alignment padding of the plane buffer was written" % name


def _unpack_arg(words, cols):
  w = np.asarray(words).view(np.uint32)
  return ((w[:, :, None] >> (2 * np.arange(16, dtype=np.uint32))) & 3).reshape(w.shape[0], cols).astype(np.int64)


# ------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------

def _patches(x):
  """x [B, H, W, C] -> padded image [B, H+2, W+2, C] and im2col [B, H, W, 9C] in (ky, kx, c) order"""
  B, H, W, C = x.shape
  xp = np.zeros((B, H + 2, W + 2, C), np.float64)
  xp[:, 1:-1, 1:-1] = x
  cols = [xp[:, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)]
  return xp, np.concatenate(cols, axis=3)


def _ref_fwd(x, k, bias):
  """conv values per pooled window v4 [B, P*F, 4] (pos = 2 dy + dx), sum |b| + sum|x||w| of each (s4)"""
  B, H, W, C = x.shape
  F = k.shape[3]
  _, pt = _patches(x)
  km = k.astype(np.float64).reshape(9 * C, F)
  conv = pt @ km + bias.astype(np.float64)
  absn = np.abs(pt) @ np.abs(km) + np.abs(bias.astype(np.float64))

  def win(a):
    a = a.reshape(B, H // 2, 2, W // 2, 2, F).transpose(0, 1, 3, 5, 2, 4)
    return a.reshape(B, (H // 2) * (W // 2) * F, 4)
  return win(conv), win(absn)


def _fwd_bound(path, C, s4):
  """componentwise bound of each conv value
     SIMT:  bias, then an FMA chain of n = 9C -> gamma(9C) (|b| + sum|x||w|)
     wgmma: 3xTF32 drops a_lo b_lo and the residuals of both splits: <= 3.001 * 2^-22 sum|x||w| (s4 also holds |b|,
            which only loosens it); the MMAs accumulate 3 * 16C products of the 4x4xC patch (zeros of W' included)
            and the bias is added once.  Tensor-core fp32 accumulation is not guaranteed to round to nearest, so the
            accumulation term ASSUMES u = 2^-23 per addition: gamma_23(48C + 1) * 1.002 (|b| + sum|x||w|) (the 1.002
            covers the three split products' magnitudes against |x||w|)."""
  if path == "simt":
    return _gamma(9 * C) * s4
  return 3.001 * 2.0 ** -22 * s4 + _gamma(48 * C + 1, 2.0 ** -23) * 1.002 * s4


def _fwd_checks(where, label, f16, v4, e4, vals, bits, arg):
  """pooled values, sign bits and arg-max of one forward against the fp64 windows (v4) and their bounds (e4)"""
  smax = v4.max(axis=2)
  ref = np.maximum(smax, 0.0)
  ep = e4.max(axis=2)                       # max and ReLU are 1-Lipschitz
  plane = 2.0 ** -22 * (ref + ep) + (2.0 ** -36 if f16 else 0.0)
  _check(where + ": pooled " + label, vals, ref, ep + plane)
  sure = np.abs(smax) > ep
  bad = sure & (bits != (smax > 0))
  assert not bad.any(), "%s: %d sign bits disagree with a clear reference sign" % (where, int(bad.sum()))
  adm = v4 + e4 >= (v4 - e4).max(axis=2, keepdims=True)        # positions that may be the maximum
  ok = np.take_along_axis(adm, arg[..., None], axis=2)[..., 0]
  assert ok.all(), "%s: %d arg-max positions outside the admissible set" % (where, int((~ok).sum()))
  unique = adm.sum(axis=2) == 1
  want = np.argmax(adm, axis=2)
  bad = unique & (arg != want)
  assert not bad.any(), "%s: %d arg-max differ where the maximum is unambiguous" % (where, int(bad.sum()))


def _ref_bwd(xp, arg, g, H, W, F):
  """dk [9C*F] and db [F] routed by the kernel's arg-max, with sum|patch||g| per dk element"""
  B = xp.shape[0]
  C = xp.shape[3]
  PH, PW = H // 2, W // 2
  a = arg.reshape(B, PH, PW, F)
  gg = g.astype(np.float64).reshape(B, PH, PW, F)
  dk = np.zeros((3, 3, C, F))
  ak = np.zeros((3, 3, C, F))
  for pos in range(4):
    dy, dx = pos >> 1, pos & 1
    gp = np.where(a == pos, gg, 0.0)
    for ky in range(3):
      for kx in range(3):
        y0, x0 = dy + ky, dx + kx
        tap = xp[:, y0:y0 + 2 * PH:2, x0:x0 + 2 * PW:2, :]        # [B, PH, PW, C]
        dk[ky, kx] += np.einsum("bhwc,bhwf->cf", tap, gp)
        ak[ky, kx] += np.einsum("bhwc,bhwf->cf", np.abs(tap), np.abs(gp))
  return dk.reshape(-1), gg.sum(axis=(0, 1, 2)), ak.reshape(-1), np.abs(gg).sum(axis=(0, 1, 2))


def _bwd_chain(B, H, W, C, F, sms):
  """longest rounding chain of one dk / db element: a thread FMAs over its ceil(B / grid) images x PH rows x
  ceil(PW / G) pixels, then the G-group sum, then conv_stem_reduce_kernel's lane stride over the grid = min(B, 4 SMs)
  partials (ceil(grid / 32)) and the 5-step shuffle tree."""
  PH, PW = H // 2, W // 2
  grid = min(B, 4 * sms)
  G = _simt_groups(C, F)
  return -(-B // grid) * PH * -(-PW // G) + G + -(-grid // 32) + 5


# ------------------------------------------------------------------------------------------------------------------
# calls
# ------------------------------------------------------------------------------------------------------------------

def _fwd(torch, _lib, lib, monkeypatch, path, xd, kd, bd, B, H, W, C, F):
  """runs the forward into guarded buffers; checks guards, padding; returns (planes buffer, layout, arg words)"""
  monkeypatch.setenv("ADN_CONV_PATH", path)
  cols = (H // 2) * (W // 2) * F
  L = _Layout(_lib.plane_format() == _lib.PLANES_F16, B, cols)
  assert L.bytes == _lib.query(_lib.Q_PLANES_BYTES, B, cols)
  planes = _alloc(torch, L.bytes)
  arg = _alloc(torch, B * cols // 16 * 4, SENTINEL)
  _lib.check(lib.adn_conv_stem_fwd(xd.data_ptr(), kd.data_ptr(), bd.data_ptr(), planes.data_ptr(), arg.data_ptr(), B,
                                   H, W, C, F, _sp(torch)), "adn_conv_stem_fwd")
  where = "%s %dx%dx%d F%d B%d" % (path, H, W, C, F, B)
  _guard_ok(where + " planes", planes, L.bytes)
  _guard_ok(where + " argmax", arg, B * cols // 16 * 4)
  return planes, L, arg[:B * cols // 16 * 4].view(torch.int32).view(B, cols // 16)


def _bwd(torch, _lib, lib, xd, argw, gd, B, H, W, C, F):
  ws_bytes = _lib.query(_lib.Q_CONV_STEM_BWD_WS, B, C, F)
  ws = _alloc(torch, ws_bytes, SENTINEL)
  nk = 9 * C * F
  dk = _alloc(torch, 4 * nk, SENTINEL)
  db = _alloc(torch, 4 * F, SENTINEL)
  _lib.check(lib.adn_conv_stem_bwd(xd.data_ptr(), argw.data_ptr(), gd.data_ptr(), dk.data_ptr(), db.data_ptr(), B, H, W,
                                   C, F, ws.data_ptr(), ws_bytes, _sp(torch)), "adn_conv_stem_bwd")
  where = "bwd %dx%dx%d F%d B%d" % (H, W, C, F, B)
  _guard_ok(where + " workspace", ws, ws_bytes)
  _guard_ok(where + " dkernel", dk, 4 * nk)
  _guard_ok(where + " dbias", db, 4 * F)
  return dk[:4 * nk].view(torch.float32), db[:4 * F].view(torch.float32)


def _fwd_paths(H, W, C, F):
  return ["simt"] + (["tc"] if _tc_fwd_supported(H, W, C, F) else [])


def _run_random(torch, _lib, lib, monkeypatch, f16, B, H, W, C, F, seed):
  """random data: every forward path and the backward against the fp64 bounds; determinism of both"""
  rng = np.random.default_rng(seed)
  x = rng.uniform(0, 1, (B, H, W, C)).astype(F32)
  x[::2] -= 0.5                                   # some signed images as well
  k = (rng.standard_normal((3, 3, C, F)) * np.sqrt(2.0 / (9 * C))).astype(F32)
  bias = (rng.standard_normal(F) * 0.1).astype(F32)
  v4, s4 = _ref_fwd(x, k, bias)
  xd, kd, bd = (torch.as_tensor(a).cuda() for a in (x, k, bias))
  cols = (H // 2) * (W // 2) * F
  outs = {}
  for path in _fwd_paths(H, W, C, F):
    planes, L, argw = _fwd(torch, _lib, lib, monkeypatch, path, xd, kd, bd, B, H, W, C, F)
    where = "%s %dx%dx%d F%d B%d" % (path, H, W, C, F, B)
    _padding_ok(where, torch, planes, L)
    vals, bits = _decode(torch, planes, L)
    arg = _unpack_arg(argw.cpu().numpy(), cols)
    _fwd_checks(where, "simt" if path == "simt" else "wgmma", f16, v4, _fwd_bound(path, C, s4), vals[:, :cols], bits[:, :cols], arg)
    again, _, argw2 = _fwd(torch, _lib, lib, monkeypatch, path, xd, kd, bd, B, H, W, C, F)
    assert torch.equal(again, planes) and torch.equal(argw2, argw), "%s: two forward calls differ" % where
    outs[path] = (vals[:, :cols], argw, arg)
  # backward from the SIMT forward's routing, gradient masked by its own pooled > 0
  vals, argw, arg = outs["simt"]
  g = (rng.standard_normal((B, cols)) / B).astype(F32)
  g = np.where(vals > 0, g, F32(0))
  gd = torch.as_tensor(g).cuda()
  xp, _ = _patches(x)
  dk_ref, db_ref, ak, ab = _ref_bwd(xp, arg, g, H, W, F)
  dk, db = _bwd(torch, _lib, lib, xd, argw, gd, B, H, W, C, F)
  dk2, db2 = _bwd(torch, _lib, lib, xd, argw, gd, B, H, W, C, F)
  where = "bwd %dx%dx%d F%d B%d" % (H, W, C, F, B)
  assert torch.equal(dk, dk2) and torch.equal(db, db2), "%s: two backward calls differ" % where
  n = _bwd_chain(B, H, W, C, F, _sms(_lib))
  _check(where + ": dkernel simt", dk.cpu().numpy(), dk_ref, _gamma(n) * 1.002 * ak)
  _check(where + ": dbias simt", db.cpu().numpy(), db_ref, _gamma(n) * ab)


# ------------------------------------------------------------------------------------------------------------------
# A. exact dyadic data: every kernel bit-exact
# ------------------------------------------------------------------------------------------------------------------

EXACT = [(4, 16, 16, 1, 16), (3, 10, 26, 3, 16), (2, 16, 32, 1, 32), (3, 6, 86, 3, 32), (2, 28, 28, 1, 48),
         (2, 32, 32, 3, 64), (1, 6, 4, 3, 48), (5, 2, 2, 1, 64)]


@pytest.mark.parametrize("B,H,W,C,F", EXACT)
def test_conv_stem_exact(env, monkeypatch, B, H, W, C, F):
  """x in {0, 1/2, 1}, w in {-1/8, 0, 1/8}, bias n/64, g = j/128 (7 significant bits): every product and partial sum
  is a multiple of its quantum below 2^24 quanta, and every operand splits into TF32 with lo = 0, so every kernel is
  exact in any order.  The planes must be byte-identical to adn_planes_split of the exact pooled values, every sign
  bit and every arg-max (first maximum in scan order, decided here by many exact ties) exact, and dkernel / dbias of
  the backward byte-identical to the exact sums."""
  torch, _lib, lib, f16 = env
  rng = np.random.default_rng(1000 + B * H * W * C + F)
  x = (rng.integers(0, 3, (B, H, W, C)) / 2.0).astype(F32)
  k = (rng.integers(-1, 2, (3, 3, C, F)) / 8.0).astype(F32)
  bias = (rng.integers(-8, 9, F) / 64.0).astype(F32)
  v4, s4 = _ref_fwd(x, k, bias)
  # the bit budget: quantum of x w and b is 2^-4 * 2^-6 = 2^-10 (x on k/16, w on m/64, b on n/64)
  assert (s4 / 2.0 ** -10).max() < 2 ** 24
  ref = np.maximum(v4.max(axis=2), 0.0)
  want_arg = np.argmax(v4, axis=2)                       # first maximum in (dy, dx) scan order
  ties = ((v4 == v4.max(axis=2, keepdims=True)).sum(axis=2) > 1) & (ref > 0)
  assert ties.sum() >= max(8, ref.size // 100), "too few exact ties between positive window maxima: %d" % ties.sum()
  cols = (H // 2) * (W // 2) * F
  xd, kd, bd = (torch.as_tensor(a).cuda() for a in (x, k, bias))
  want_planes = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, cols),), dtype=torch.uint8, device="cuda")
  refd = torch.as_tensor(ref.astype(F32)).cuda()
  assert np.array_equal(refd.cpu().numpy().astype(np.float64), ref)
  _lib.check(lib.adn_planes_split(refd.data_ptr(), B, cols, want_planes.data_ptr(), _sp(torch)), "adn_planes_split")
  argw = None
  for path in _fwd_paths(H, W, C, F):
    planes, L, aw = _fwd(torch, _lib, lib, monkeypatch, path, xd, kd, bd, B, H, W, C, F)
    where = "exact %s %dx%dx%d F%d B%d" % (path, H, W, C, F, B)
    got = planes[:L.bytes]
    if not torch.equal(got, want_planes):
      d = (got != want_planes).nonzero()[:4].flatten().tolist()
      raise AssertionError("%s: planes differ from adn_planes_split of the exact values at bytes %s" % (where, d))
    _, bits = _decode(torch, planes, L)
    assert np.array_equal(bits[:, :cols], ref > 0), where + ": sign bits"
    arg = _unpack_arg(aw.cpu().numpy(), cols)
    bad = arg != want_arg
    assert not bad.any(), "%s: %d arg-max are not the first maximum (%d at ties)" % (where, bad.sum(), (bad & ties).sum())
    if argw is None:
      argw = aw
    else:
      assert torch.equal(aw, argw), where + ": arg-max words differ between the paths"
  g = (rng.integers(-127, 128, (B, cols)) / 128.0)
  g = np.where(ref > 0, g, 0.0).astype(F32)
  xp, _ = _patches(x)
  dk_ref, db_ref, ak, ab = _ref_bwd(xp, want_arg, g, H, W, F)
  # quantum of x g is 2^-4 * 2^-7 = 2^-11, of g alone 2^-7
  assert (ak / 2.0 ** -11).max() < 2 ** 24 and (ab / 2.0 ** -7).max() < 2 ** 24
  gd = torch.as_tensor(g).cuda()
  want_dk, want_db = dk_ref.astype(F32), db_ref.astype(F32)
  assert np.array_equal(want_dk.astype(np.float64), dk_ref) and np.array_equal(want_db.astype(np.float64), db_ref)
  dk, db = _bwd(torch, _lib, lib, xd, argw, gd, B, H, W, C, F)
  where = "exact bwd %dx%dx%d F%d B%d" % (H, W, C, F, B)
  assert np.array_equal(dk.cpu().numpy().view(np.uint32), want_dk.view(np.uint32)), where + ": dkernel"
  assert np.array_equal(db.cpu().numpy().view(np.uint32), want_db.view(np.uint32)), where + ": dbias"


# ------------------------------------------------------------------------------------------------------------------
# B / C. random data at the shapes and batches where the kernels change behaviour
# ------------------------------------------------------------------------------------------------------------------

_CF = [(c, f) for c in (1, 3) for f in (16, 32, 48, 64)]
# (H, W, B): P = 1; non-square; P = 64, 65, 128, 129 around the 128-row forward tiles and 64-pixel backward tiles
_SMALL = [(2, 2, 1), (6, 4, 3), (36, 20, 2), (16, 16, 2), (10, 26, 3), (16, 32, 2), (6, 86, 2)]
SHAPES = [(B, H, W, C, F) for (C, F) in _CF for (H, W, B) in _SMALL]


@pytest.mark.parametrize("B,H,W,C,F", SHAPES)
def test_conv_stem_random(env, monkeypatch, B, H, W, C, F):
  torch, _lib, lib, f16 = env
  _run_random(torch, _lib, lib, monkeypatch, f16, B, H, W, C, F, seed=B * 131 + H * 7 + W + C * 3 + F)


@pytest.mark.parametrize("batch", ["1", "sms-1", "4sms+1"])
@pytest.mark.parametrize("C,F", _CF)
def test_conv_stem_batches(env, monkeypatch, batch, C, F):
  """28x28x1 / 32x32x3 at batch 1, one below the SM count, and one above 4 SMs (several images per SIMT backward CTA,
  the 4-deep image ring of the F = 16 wgmma forward wraps)"""
  torch, _lib, lib, f16 = env
  sms = _sms(_lib)
  B = {"1": 1, "sms-1": sms - 1, "4sms+1": 4 * sms + 1}[batch]
  H = W = 28 if C == 1 else 32
  _run_random(torch, _lib, lib, monkeypatch, f16, B, H, W, C, F, seed=B + C * 10 + F)


def _boundary_shapes():
  out = []
  for C in (1, 3):
    for F in (16, 32):
      h = _largest_square(C, F, _tc_fwd_supported)
      out += [(2, h, h, C, F), (2, h + 2, h + 2, C, F)]    # last wgmma-forward square, first SIMT fall-back
  return out + [(2, 152, 152, 1, F) for F in (16, 32, 48, 64)] + [(2, 86, 86, 3, F) for F in (16, 32, 48, 64)]


@pytest.mark.parametrize("B,H,W,C,F", _boundary_shapes())
def test_conv_stem_large_images(env, monkeypatch, B, H, W, C, F):
  """both sides of the wgmma forward's shared-memory boundary, and the envelope corners 152x152x1 / 86x86x3"""
  torch, _lib, lib, f16 = env
  assert _accepted(H, W, C, F)
  _run_random(torch, _lib, lib, monkeypatch, f16, B, H, W, C, F, seed=H * 5 + C + F)


def test_conv_stem_beyond_2g_elements(env, monkeypatch):
  """B * cols > 2^31 elements (32x32x3, F = 64, B = 140000: about 21-30 GB); reference on the first rows, the last
  rows, the rows straddling element 2^31 of the dense gradient and of the hi plane's flat index"""
  torch, _lib, lib, f16 = env
  B, H, W, C, F = 140000, 32, 32, 3, 64
  cols = (H // 2) * (W // 2) * F
  assert B * cols > 2 ** 31
  L = _Layout(f16, B, cols)
  kb = (2 ** 31 // L.bk) // B                              # k-block of the plane in which element 2^31 falls
  r31 = 2 ** 31 // L.bk - kb * B
  rows = sorted({0, 1, r31 - 1, r31, 2 ** 31 // cols - 1, 2 ** 31 // cols, B - 2, B - 1})
  free, _ = torch.cuda.mem_get_info()
  need = B * H * W * C * 4 + L.bytes + B * cols // 16 * 4 + B * cols * 4 + (1 << 30)
  if free < need:
    pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 2 ** 30, free / 2 ** 30))
  gen = torch.Generator(device="cuda").manual_seed(7)
  xd = torch.rand((B, H, W, C), device="cuda", generator=gen)
  rng = np.random.default_rng(7)
  k = (rng.standard_normal((3, 3, C, F)) * np.sqrt(2.0 / (9 * C))).astype(F32)
  bias = (rng.standard_normal(F) * 0.1).astype(F32)
  kd, bd = torch.as_tensor(k).cuda(), torch.as_tensor(bias).cuda()
  try:
    planes, L2, argw = _fwd(torch, _lib, lib, monkeypatch, "simt", xd, kd, bd, B, H, W, C, F)
    x = xd[torch.as_tensor(rows, device="cuda")].cpu().numpy()
    v4, s4 = _ref_fwd(x, k, bias)
    vals, bits = _decode(torch, planes, L2, rows)
    del planes
    arg = _unpack_arg(argw[torch.as_tensor(rows, device="cuda")].cpu().numpy(), cols)
    _fwd_checks("2G", "simt", f16, v4, _fwd_bound("simt", C, s4), vals[:, :cols], bits[:, :cols], arg)
    # backward: gradient only on the checked rows, so their sum is the reference
    g = (rng.standard_normal((len(rows), cols)) / len(rows)).astype(F32)
    g = np.where(vals[:, :cols] > 0, g, F32(0))
    gd = torch.zeros((B, cols), dtype=torch.float32, device="cuda")
    gd[torch.as_tensor(rows, device="cuda")] = torch.as_tensor(g).cuda()
    xp, _ = _patches(x)
    dk_ref, db_ref, ak, ab = _ref_bwd(xp, arg, g, H, W, F)
    dk, db = _bwd(torch, _lib, lib, xd, argw, gd, B, H, W, C, F)
    n = _bwd_chain(B, H, W, C, F, _sms(_lib))
    _check("2G bwd: dkernel simt", dk.cpu().numpy(), dk_ref, _gamma(n) * ak)
    _check("2G bwd: dbias simt", db.cpu().numpy(), db_ref, _gamma(n) * ab)
  finally:
    del xd
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# D. contract checks
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("path", ["simt", "tc"])
def test_conv_stem_overflow_flag(env, monkeypatch, path):
  """fp16 planes: a pooled value >= 65520 raises adn_plane_overflow on both forward paths, 65519 does not; TF32
  planes never raise it"""
  torch, _lib, lib, f16 = env
  B, H, W, C, F = 3, 8, 8, 1, 16
  assert path == "simt" or _tc_fwd_supported(H, W, C, F)
  x = np.ones((B, H, W, C), F32)
  k = np.zeros((3, 3, C, F), F32)
  xd, kd = torch.as_tensor(x).cuda(), torch.as_tensor(k).cuda()
  for top, raises in ((65519.0, False), (65520.0, f16), (1e30, f16)):
    bias = np.zeros(F, F32)
    bias[5] = top
    bd = torch.as_tensor(bias).cuda()
    _lib.plane_overflow()
    _fwd(torch, _lib, lib, monkeypatch, path, xd, kd, bd, B, H, W, C, F)
    assert _lib.plane_overflow(_sp(torch)) == raises, "%s: pooled maximum %r" % (path, top)


def _envelope_shapes():
  out = [(64, 64, 3, 16), (96, 96, 1, 16), (48, 48, 3, 64), (28, 28, 1, 64), (32, 32, 3, 64), (44, 44, 3, 16),
         (46, 46, 3, 16), (100, 100, 1, 16), (102, 102, 1, 16)]
  for C in (1, 3):
    for F in (16, 32, 48, 64):
      h = _largest_square(C, F, lambda *a: True)
      out.append((h, h, C, F))                                  # 154 (C = 1) / 88 (C = 3)
      hb = _largest_square(C, F, _simt_bwd_staged)
      out += [(hb, hb, C, F), (hb + 2, hb + 2, C, F)]           # last staged / first image-only SIMT backward
  out += [(152, 152, 1, 16), (86, 86, 3, 64), (2, 6142, 1, 64), (6142, 2, 1, 16), (2, 2046, 3, 16), (2046, 2, 3, 48)]
  return sorted(set(out))


@pytest.mark.parametrize("fwd_path", ["simt", "tcgen05"])
@pytest.mark.parametrize("H,W,C,F", _envelope_shapes())
def test_conv_stem_envelope(env, monkeypatch, fwd_path, H, W, C, F):
  """every shape the forward accepts, the backward accepts, routed by the arg-max words of either forward path
  (ADN_CONV_PATH=simt, or the default wgmma forward, which falls back to SIMT where it does not fit); and the result
  is right"""
  torch, _lib, lib, f16 = env
  assert _accepted(H, W, C, F)
  B = 2
  rng = np.random.default_rng(H * 3 + W + C + F)
  x = rng.uniform(0, 1, (B, H, W, C)).astype(F32)
  k = (rng.standard_normal((3, 3, C, F)) * np.sqrt(2.0 / (9 * C))).astype(F32)
  bias = (rng.standard_normal(F) * 0.1).astype(F32)
  xd, kd, bd = (torch.as_tensor(a).cuda() for a in (x, k, bias))
  cols = (H // 2) * (W // 2) * F
  planes, L, argw = _fwd(torch, _lib, lib, monkeypatch, fwd_path, xd, kd, bd, B, H, W, C, F)
  vals, _ = _decode(torch, planes, L)
  vals = vals[:, :cols]
  arg = _unpack_arg(argw.cpu().numpy(), cols)
  g = np.where(vals > 0, rng.standard_normal((B, cols)) / B, 0.0).astype(F32)
  gd = torch.as_tensor(g).cuda()
  dk, db = _bwd(torch, _lib, lib, xd, argw, gd, B, H, W, C, F)
  xp, _ = _patches(x)
  dk_ref, db_ref, ak, ab = _ref_bwd(xp, arg, g, H, W, F)
  n = _bwd_chain(B, H, W, C, F, _sms(_lib))
  _check("envelope: dkernel simt", dk.cpu().numpy(), dk_ref, _gamma(n) * 1.002 * ak)
  _check("envelope: dbias simt", db.cpu().numpy(), db_ref, _gamma(n) * ab)


@pytest.mark.parametrize("H,W,C,F", [(156, 156, 1, 16), (90, 90, 3, 64), (2, 6144, 1, 16), (2048, 2, 3, 32),
                                     (7, 8, 1, 16), (8, 8, 2, 16), (8, 8, 1, 24)])
def test_conv_stem_rejects_outside_envelope(env, monkeypatch, H, W, C, F):
  torch, _lib, lib, f16 = env
  t = torch.zeros((1 << 16,), dtype=torch.float32, device="cuda")
  p = t.data_ptr()
  assert not _accepted(H, W, C, F)
  want = ERR_INVALID if (H % 2 or W % 2) else ERR_UNSUPPORTED
  for fwd_path in ("tc", "simt"):
    monkeypatch.setenv("ADN_CONV_PATH", fwd_path)
    assert lib.adn_conv_stem_fwd(p, p, p, p, p, 2, H, W, C, F, _sp(torch)) == want
    assert lib.adn_conv_stem_bwd(p, p, p, p, p, 2, H, W, C, F, p, 1 << 18, _sp(torch)) == want
  assert (t == 0).all()
