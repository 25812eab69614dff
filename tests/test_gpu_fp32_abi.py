"""GPU tests of the library's fp32 row-major boundary, element by element against float64 NumPy:

  a. non-finite values through every plane writer (split, GEMM epilogues, head dlogits planes, optimizer plane refresh,
     the conv stem's TF32 operand staging), in both plane formats;
  b. adn_planes_split / _scaled / adn_planes_merge at the value edges of both formats, restated in NumPy bit for bit;
  c. the fp32 dense ABI (adn_dense_fwd / adn_dense_bwd) on PATH_SIMT, PATH_AUTO and PATH_TCGEN05, with its path
     choice and workspace errors;
  d. adn_colsum.

Bounds are componentwise.  Where a kernel sums sequentially the bound is gamma(n) * sum|terms| with
gamma(n) = n u / (1 - n u), u = 2^-24, and n the longest rounding chain in the kernel's order (written beside each
bound).  The tensor-core paths use 3e-6 * (|A| |B|)_ij.  Every output and workspace is filled with NaN before a call,
so an element that was never written shows up.
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TOL = 3e-6
F32, F16 = np.float32, np.float16
ERR_INVALID, ERR_UNSUPPORTED, ERR_WORKSPACE = -22, -95, -12

# bit patterns of the non-finite values: the canonical NaN of GPU arithmetic (0x7FFFFFFF) and its negative, NumPy's
# quiet NaNs, a signalling NaN, a NaN whose low 13 bits are clear, and +-Inf
NONFINITE = [0x7FFFFFFF, 0xFFFFFFFF, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFF000, 0x7F800000, 0xFF800000]

_WORST = {}    # check name -> largest |err| / bound seen in this module (printed at teardown, pytest -s)


def _gamma(n):
  return n * U / (1.0 - n * U)


def _gbound(n, terms):
  """gamma(n) * sum|terms|, plus n * 2^-150 for the roundings of subnormal partial sums"""
  return _gamma(n) * terms + n * 2.0 ** -150


def _check(name, got, ref, bound):
  """|got - ref| <= bound element by element"""
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


def _open():
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  return torch, _lib, lib


@pytest.fixture(scope="module", params=["f16", "tf32"])
def env(request):
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _lib.set_plane_format(_lib.PLANES_F16 if request.param == "f16" else _lib.PLANES_TF32)
  _lib.plane_overflow()      # clear the sticky flag
  yield torch, _lib, lib
  _lib.set_plane_format(before)


@pytest.fixture(scope="module")
def gpu():
  """the fp32 ABI does not depend on the process plane format (its tensor path always uses TF32 planes)"""
  torch, _lib, lib = _open()
  yield torch, _lib, lib
  _lib.set_dense_path(_lib.PATH_AUTO)


def _sp(torch):
  return torch.cuda.current_stream().cuda_stream


def _dev(torch, a):
  return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _nan(torch, *shape):
  return torch.full(shape, float("nan"), device="cuda")


def _bytes(t):
  import torch
  return t.reshape(-1).view(torch.uint8).cpu().numpy().copy()


def _from_bits(bits):
  return np.asarray(bits, dtype=np.uint64).astype(np.uint32).view(F32)


# ------------------------------------------------------------------------------------------------------------------
# the two plane formats restated in NumPy (plane_fmt.cuh)
# ------------------------------------------------------------------------------------------------------------------

def _rna(a):
  """cvt.rna.tf32 as the kernels emulate it: add half a TF32 ulp to the bit pattern, clear the low 13 bits"""
  u = np.asarray(a, dtype=F32).view(np.uint32).astype(np.uint64)
  return (((u + 0x1000) & 0xFFFFE000) & 0xFFFFFFFF).astype(np.uint32).view(F32)


def _split_tf32(sv):
  with np.errstate(all="ignore"):
    hi = _rna(sv)
    lo = _rna((sv - hi).astype(F32))
  nf = ~np.isfinite(sv)
  hi = np.where(nf, sv, hi).astype(F32)
  lo = np.where(nf, F32(0), lo).astype(F32)
  return hi, lo


def _split_f16(sv):
  with np.errstate(all="ignore"):
    hi = sv.astype(F16)
    lo = ((sv - hi.astype(F32)).astype(F32) * F32(2048)).astype(F16)
  return hi, lo


def _merge_np(hi, lo, f16):
  with np.errstate(all="ignore"):
    if f16:
      return (hi.astype(F32) + lo.astype(F32) * F32(2.0 ** -11)).astype(F32)
    return (hi + lo).astype(F32)


class _Layout:
  """byte layout of a plane tensor [rows, cols]: hi plane, lo plane ([nkb][rows][BK] + alignment tail), sign bits"""

  def __init__(self, f16, rows, cols):
    self.f16, self.rows, self.cols = f16, rows, cols
    self.bk, self.es = (64, 2) if f16 else (32, 4)
    self.nkb = -(-cols // self.bk)
    self.n = self.nkb * rows * self.bk
    self.elems = -(-self.n // 128) * 128
    self.nb32 = self.nkb * self.bk // 32
    self.bits_off = 2 * self.elems * self.es
    self.bytes = self.bits_off + (-(-(rows * self.nb32) // 64) * 64) * 4

  def planes(self, raw):
    """(hi, lo) as [rows, nkb * BK] arrays of fp16 / fp32, and the sign-bit words [nb32][rows]"""
    dt = F16 if self.f16 else F32
    def one(off):
      p = raw[off: off + self.n * self.es].view(dt).reshape(self.nkb, self.rows, self.bk)
      return p.transpose(1, 0, 2).reshape(self.rows, self.nkb * self.bk)
    bits = raw[self.bits_off: self.bits_off + self.nb32 * self.rows * 4].view(np.uint32).reshape(self.nb32, self.rows)
    return one(0), one(self.elems * self.es), bits

  def want(self, sv):
    """what the split must write for the scaled values sv [rows, cols]: hi, lo (padded) and sign-bit words"""
    pad = np.zeros((self.rows, self.nkb * self.bk), dtype=F32)
    pad[:, :self.cols] = sv
    hi, lo = _split_f16(pad) if self.f16 else _split_tf32(pad)
    pos = (pad > 0).reshape(self.rows, self.nb32, 32).astype(np.uint64)
    bits = (pos << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32).T
    return hi, lo, bits


def _split(torch, _lib, lib, src, rows, cols, s=0, fill=0xFF, offset=0):
  """adn_planes_split_scaled of the device tensor src (from `offset` bytes on) into a buffer pre-filled with `fill`;
  returns (rc, uint8 tensor)"""
  out = torch.full((_lib.query(_lib.Q_PLANES_BYTES, rows, cols),), fill, dtype=torch.uint8, device="cuda")
  rc = lib.adn_planes_split_scaled(src.data_ptr() + offset, rows, cols, out.data_ptr(), s, _sp(torch))
  return rc, out


def _merge(torch, _lib, lib, planes, rows, cols):
  out = _nan(torch, rows, cols)
  _lib.check(lib.adn_planes_merge(planes.data_ptr(), rows, cols, out.data_ptr(), _sp(torch)), "merge")
  return out.cpu().numpy()


def _same_bits(name, got, want):
  """bit-identical, except that a zero is compared as a number (the sign of zero is not part of the contract)"""
  gb = got.view(np.uint16 if got.dtype == F16 else np.uint32)
  wb = want.view(np.uint16 if want.dtype == F16 else np.uint32)
  ok = (gb == wb) | ((want == 0) & (got == 0))
  if not ok.all():
    i = np.unravel_index(np.argmin(ok), ok.shape)
    raise AssertionError("%s: %d elements differ; at %s got 0x%x want 0x%x" % (name, int((~ok).sum()), i, gb[i], wb[i]))


def _nonfinite_mask_eq(name, got, want):
  g, w = ~np.isfinite(got), ~np.isfinite(want)
  if not np.array_equal(g, w):
    i = np.unravel_index(np.argmax(g != w), g.shape)
    raise AssertionError("%s: non-finite mask differs in %d elements; at %s got %r want %r"
                         % (name, int((g != w).sum()), i, got[i], want[i]))


# ------------------------------------------------------------------------------------------------------------------
# a. non-finite values through every plane writer
# ------------------------------------------------------------------------------------------------------------------

def test_nonfinite_split_merge(env):
  torch, _lib, lib = env
  f16 = _lib.plane_format() == _lib.PLANES_F16
  dev_nan = (torch.zeros(1, device="cuda") / 0).view(torch.int32).item() & 0xFFFFFFFF
  print("\nNaN made by the device (0 / 0): 0x%08X" % dev_nan)
  R, C = 4, 40
  rng = np.random.default_rng(11)
  clean = rng.standard_normal((R, C)).astype(F32)
  a = clean.copy()
  at = [(k % R, (7 * k + 3) % C) for k in range(len(NONFINITE))]
  for (r, c), b in zip(at, NONFINITE):
    a[r, c] = _from_bits([b])[0]
  L = _Layout(f16, R, C)
  cd, ad = _dev(torch, clean), _dev(torch, a)
  for s in (0, 5):
    rc, pc = _split(torch, _lib, lib, cd, R, C, s)
    _lib.check(rc, "split")
    rc, pa = _split(torch, _lib, lib, ad, R, C, s)
    _lib.check(rc, "split")
    assert not _lib.plane_overflow(), "a non-finite value raised the fp16 overflow flag"
    back, back_c = _merge(torch, _lib, lib, pa, R, C), _merge(torch, _lib, lib, pc, R, C)
    fin = np.isfinite(a)
    assert np.array_equal(back[fin].view(np.uint32), back_c[fin].view(np.uint32)), "finite neighbours changed"
    hi, lo, bits = L.planes(_bytes(pa))
    hic, loc, bitsc = L.planes(_bytes(pc))
    assert np.array_equal(hi[:, :C][fin].view(np.uint8), hic[:, :C][fin].view(np.uint8))
    assert np.array_equal(lo[:, :C][fin].view(np.uint8), loc[:, :C][fin].view(np.uint8))
    for (r, c), b in zip(at, NONFINITE):
      v = _from_bits([b])[0]
      where = "s=%d 0x%08X" % (s, b)
      if np.isnan(v):
        assert np.isnan(back[r, c]), "%s merged to %r" % (where, back[r, c])
        assert np.isnan(hi[r, c]), "%s: hi plane %r" % (where, hi[r, c])
      elif f16:
        assert not np.isfinite(back[r, c]), where
        assert hi[r, c] == v, where
      else:
        assert back[r, c] == v, "%s merged to %r" % (where, back[r, c])
        assert hi[r, c] == v and lo[r, c] == 0, where
      # sign bit: NaN is not > 0
      assert bool((bits[c // 32, r] >> (c % 32)) & 1) == bool(v > 0), where


def _inject(rng, a, n_at, patterns=NONFINITE):
  """puts the patterns into a at distinct random positions"""
  flat = rng.choice(a.size, size=n_at, replace=False)
  for i, b in zip(flat, patterns * (n_at // len(patterns) + 1)):
    a.reshape(-1)[i] = _from_bits([b])[0]


NANS = [b for b in NONFINITE if np.isnan(_from_bits([b])[0])]


@pytest.mark.parametrize("where", ["x", "w", "dz"])
@pytest.mark.parametrize("act", [0, 1])
def test_nonfinite_dense_planes(env, where, act):
  """The non-finite masks of every output of adn_dense_fwd_p / adn_dense_bwd_p equal those of the SIMT fp32 path on
  the same inputs.  With ReLU, SIMT's relu(NaN) = 0 (fmaxf) is the reference; the backward masks by x > 0.
  Under ReLU the forward operands carry NaNs only: an Inf operand meets its partner's lo plane on the plane path
  (Inf * 0, or Inf - Inf when hi and lo differ in sign), so a sum that is +Inf on SIMT can be NaN there, and ReLU maps
  the two to Inf and 0.  Without ReLU both are non-finite."""
  torch, _lib, lib = env
  B, I, O = 130, 40, 70
  rng = np.random.default_rng(100 + act + 3 * len(where))
  x = rng.standard_normal((B, I)).astype(F32)
  w = (rng.standard_normal((I, O)) / np.sqrt(I)).astype(F32)
  dz = rng.standard_normal((B, O)).astype(F32)
  b = rng.standard_normal(O).astype(F32)
  _inject(rng, {"x": x, "w": w, "dz": dz}[where], 8, NANS if act and where != "dz" else NONFINITE)
  xd, wd, dzd, bd = (_dev(torch, t) for t in (x, w, dz, b))
  sp = _sp(torch)
  # SIMT fp32 reference of the masks
  _lib.set_dense_path(_lib.PATH_SIMT)
  try:
    y_s, dx_s, dw_s, db_s = _nan(torch, B, O), _nan(torch, B, I), _nan(torch, I, O), _nan(torch, O)
    _lib.check(lib.adn_dense_fwd(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), y_s.data_ptr(), B, I, O, act, None, 0, sp),
               "simt fwd")
    wsb = _lib.query(_lib.Q_DENSE_BWD_WS, B, I, O)
    ws = torch.empty((wsb,), dtype=torch.uint8, device="cuda")
    _lib.check(lib.adn_dense_bwd(xd.data_ptr(), wd.data_ptr(), dzd.data_ptr(), dx_s.data_ptr(), dw_s.data_ptr(),
                                 db_s.data_ptr(), B, I, O, act, ws.data_ptr(), wsb, sp), "simt bwd")
  finally:
    _lib.set_dense_path(_lib.PATH_AUTO)
  y_s, dx_s, dw_s = y_s.cpu().numpy(), dx_s.cpu().numpy(), dw_s.cpu().numpy()
  cs_s = np.where(np.isfinite(dx_s).all(axis=0), 0.0, np.nan)
  # plane path
  planes = {}
  for name, t, (r, c) in (("x", xd, (B, I)), ("w", wd, (I, O)), ("dz", dzd, (B, O))):
    rc, planes[name] = _split(torch, _lib, lib, t, r, c)
    _lib.check(rc, "split " + name)
  xp, wp, dzp = planes["x"], planes["w"], planes["dz"]
  y = _nan(torch, B, O)
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), bd.data_ptr(), None, y.data_ptr(), B, I, O, act, sp), "fwd_p")
  yp = torch.full((_lib.query(_lib.Q_PLANES_BYTES, B, O),), 0xFF, dtype=torch.uint8, device="cuda")
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), bd.data_ptr(), yp.data_ptr(), None, B, I, O, act, sp), "fwd_p")
  nb = _lib.query(_lib.Q_DENSE_BWD_P_WS, B, I, O)
  wsp = torch.full((nb,), 0xFF, dtype=torch.uint8, device="cuda")
  dw, cs = _nan(torch, I, O), _nan(torch, I)
  dxp = torch.full((_lib.query(_lib.Q_PLANES_BYTES, B, I),), 0xFF, dtype=torch.uint8, device="cuda")
  _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), wp.data_ptr(), dzp.data_ptr(), dxp.data_ptr(), None, cs.data_ptr(),
                                 dw.data_ptr(), B, I, O, act, 0, wsp.data_ptr(), nb, sp), "bwd_p")
  dx = _nan(torch, B, I)
  _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), wp.data_ptr(), dzp.data_ptr(), None, dx.data_ptr(), None, None, B, I, O,
                                 act, 0, wsp.data_ptr(), nb, sp), "bwd_p dense dx")
  _nonfinite_mask_eq("y", y.cpu().numpy(), y_s)
  _nonfinite_mask_eq("merged yp", _merge(torch, _lib, lib, yp, B, O), y_s)
  _nonfinite_mask_eq("dw", dw.cpu().numpy(), dw_s)
  _nonfinite_mask_eq("merged dxp", _merge(torch, _lib, lib, dxp, B, I), dx_s)
  _nonfinite_mask_eq("dx", dx.cpu().numpy(), dx_s)
  _nonfinite_mask_eq("dx colsum", cs.cpu().numpy(), cs_s)
  assert (~np.isfinite(y_s)).any() or (~np.isfinite(dx_s)).any() or (~np.isfinite(dw_s)).any()


def test_nonfinite_head_loss_planes(env):
  """A NaN logit makes the whole row of the merged dlogits planes NaN (softmax of a row with a NaN)."""
  torch, _lib, lib = env
  B, C, S = 130, 10, 7
  rng = np.random.default_rng(21)
  logits = rng.standard_normal((B, C)).astype(F32)
  nan_rows = [3, 40, 77, 100, 128, 129]
  for r, b in zip(nan_rows, NANS):
    logits[r, rng.integers(C)] = _from_bits([b])[0]
  labels = rng.integers(0, C, B).astype(np.int64)
  ld, lab = _dev(torch, logits), _dev(torch, labels)
  wsb = _lib.query(_lib.Q_HEAD_WS, B, C, 1)
  ws = torch.empty((wsb,), dtype=torch.uint8, device="cuda")
  loss, dl, cs = _nan(torch, 1), _nan(torch, B, C), _nan(torch, C)
  planes = torch.full((_lib.query(_lib.Q_PLANES_BYTES, B, C),), 0xFF, dtype=torch.uint8, device="cuda")
  _lib.check(lib.adn_head_loss_p(_lib.HEAD_SOFTMAX_XENT, ld.data_ptr(), lab.data_ptr(), None, loss.data_ptr(),
                                 dl.data_ptr(), planes.data_ptr(), cs.data_ptr(), S, B, C, ws.data_ptr(), wsb, _sp(torch)),
             "adn_head_loss_p")
  merged = _merge(torch, _lib, lib, planes, B, C)
  bad = np.zeros(B, dtype=bool)
  bad[nan_rows] = True
  assert np.isnan(merged[bad]).all(), "a NaN logit's dlogits planes are not all NaN"
  assert np.isfinite(merged[~bad]).all()
  assert np.isnan(dl.cpu().numpy()[bad]).all()


def test_nonfinite_opt_step_planes(env):
  """SGD with non-finite gradient elements: the refreshed weight planes hold NaN where the parameter is NaN (and +-Inf
  under TF32; fp16 planes merge +-Inf to NaN), and are byte-identical to adn_planes_split of the updated parameter."""
  torch, _lib, lib = env
  f16 = _lib.plane_format() == _lib.PLANES_F16
  R, C = 100, 70
  rng = np.random.default_rng(31)
  w = rng.standard_normal((R, C)).astype(F32)
  g = rng.standard_normal((R, C)).astype(F32)
  _inject(rng, g, 16)
  wd, gd = _dev(torch, w), _dev(torch, g)
  wp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, R, C),), dtype=torch.uint8, device="cuda")
  _lib.check(lib.adn_opt_step_p(_lib.OPT_SGD, _lib.ptr_array([wd.data_ptr()]), _lib.ptr_array([gd.data_ptr()]), None, None,
                                _lib.i64_array([R * C]), 1, _lib.f32_array([0.1]), None, _lib.ptr_array([wp.data_ptr()]),
                                _lib.i64_array([C]), _sp(torch)), "opt_step_p")
  p = wd.cpu().numpy()
  assert np.array_equal(np.isnan(p), np.isnan(g)) and np.array_equal(np.isinf(p), np.isinf(g))
  merged = _merge(torch, _lib, lib, wp, R, C)
  assert np.isnan(merged[np.isnan(p)]).all(), "the refreshed planes lost a NaN"
  assert np.array_equal(np.isfinite(merged), np.isfinite(p))
  if not f16:
    assert np.array_equal(merged[np.isinf(p)], p[np.isinf(p)])
  rc, ref = _split(torch, _lib, lib, wd, R, C, fill=0)
  _lib.check(rc, "split")
  L = _Layout(f16, R, C)
  for got, want in zip(L.planes(_bytes(wp))[:2], L.planes(_bytes(ref))[:2]):
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))


def _conv_masks(img, g, arg, H, W, C, F):
  """non-finite masks of dkernel [3,3,C,F] / dbias [F] of the SIMT backward: dK[ky,kx,c,f] sums
  patch(argmax)[ky,kx,c] * g over pooled pixels, so a non-finite pixel reaches the taps of the arg-max position only."""
  B = img.shape[0]
  PH, PW = H // 2, W // 2
  pad = np.zeros((B, H + 2, W + 2, C), dtype=bool)
  pad[:, 1:-1, 1:-1, :] = ~np.isfinite(img)
  gnf = ~np.isfinite(g.reshape(B, PH * PW, F))
  simt = np.zeros((3, 3, C, F), dtype=bool)
  for b in range(B):
    for p in range(PH * PW):
      py, px = divmod(p, PW)
      for f in range(F):
        e = p * F + f
        pos = (int(arg[b, e // 16]) >> (2 * (e % 16))) & 3
        dy, dx = pos >> 1, pos & 1
        simt[:, :, :, f] |= pad[b, 2 * py + dy: 2 * py + dy + 3, 2 * px + dx: 2 * px + dx + 3, :]
        if gnf[b, p, f]:
          simt[:, :, :, f] = True
  return simt, gnf.any(axis=(0, 1))


@pytest.mark.parametrize("case", ["pixel", "dpooled"])
def test_nonfinite_conv_stem_bwd(env, case):
  """A NaN pixel / NaN dpooled entry through the backward reaches exactly the outputs _conv_masks predicts."""
  torch, _lib, lib = env
  B, H, W, C, F = 3, 10, 10, 3, 16
  cols = (H // 2) * (W // 2) * F
  rng = np.random.default_rng(41)
  img = rng.uniform(0, 1, (B, H, W, C)).astype(F32)
  g = (rng.standard_normal((B, cols)) * 0.01).astype(F32)
  arg = rng.integers(0, 2 ** 32, (B, cols // 16), dtype=np.uint64).astype(np.uint32)
  if case == "pixel":
    img[1, 4, 5, 2] = _from_bits([0x7FFFFFFF])[0]
    img[2, 0, 9, 0] = _from_bits([0xFFFFFFFF])[0]
  else:
    g[2, 7 * F + 3] = _from_bits([0x7FFFFFFF])[0]
    g[0, 11 * F + 9] = _from_bits([0xFFFFFFFF])[0]
  simt_m, db_m = _conv_masks(img, g, arg, H, W, C, F)
  assert simt_m.any() and not simt_m.all()
  xd, gd, ad = _dev(torch, img), _dev(torch, g), _dev(torch, arg.view(np.int32))
  wsb = _lib.query(_lib.Q_CONV_STEM_BWD_WS, B, C, F)
  ws = torch.full((wsb,), 0xFF, dtype=torch.uint8, device="cuda")
  dk, db = _nan(torch, 9 * C * F), _nan(torch, F)
  _lib.check(lib.adn_conv_stem_bwd(xd.data_ptr(), ad.data_ptr(), gd.data_ptr(), dk.data_ptr(), db.data_ptr(), B, H, W,
                                   C, F, ws.data_ptr(), wsb, _sp(torch)), "adn_conv_stem_bwd")
  assert np.array_equal(~np.isfinite(dk.cpu().numpy().reshape(3, 3, C, F)), simt_m)
  assert np.array_equal(~np.isfinite(db.cpu().numpy()), db_m)


# ------------------------------------------------------------------------------------------------------------------
# b. split and merge at the value edges
# ------------------------------------------------------------------------------------------------------------------

SCALES = [-60, -15, -1, 0, 1, 7, 15, 60]
FLT_MAX = float(np.finfo(F32).max)
# scaled values sv = v * 2^s the split sees
EDGES = [float(v) for v in (
    2.0 ** -14, np.nextafter(F32(2.0 ** -14), F32(0)), np.nextafter(F32(2.0 ** -14), F32(1)), 2.0 ** -24, 2.0 ** -25,
    1.5 * 2.0 ** -25, 2.0 ** -26, 3 * 2.0 ** -27, 2.0 ** -30, 2.0 ** -40, 65504.0, 65505.0, 65519.0,
    _from_bits([0x477FEFFF])[0], _from_bits([0x477FF000])[0], 65536.0, 1.0, 1 + 2.0 ** -11, 1 + 2.0 ** -12,
    1 + 3 * 2.0 ** -12, 1 + 2.0 ** -23, 0.0, -0.0, FLT_MAX, 2.0 ** 100)]
# raw fp32 subnormal inputs (scaled by the kernel in fp32)
SUBNORMALS = [float(_from_bits([b])[0]) for b in (0x1, 0x3FF, 0x400000, 0x7FFFFF)]


def _edge_inputs(s):
  """inputs v whose scaled value hits every edge exactly (where v = edge * 2^-s is an fp32), and the subnormals"""
  vals = []
  for e in EDGES:
    for sign in (1.0, -1.0):
      v = sign * e * 2.0 ** -s
      with np.errstate(all="ignore"):
        v32 = F32(v)
        if np.isfinite(v32) and float(v32) == v and float(F32(v32 * F32(2.0 ** s))) == sign * e:
          vals.append(v32)
  vals += [F32(v) for v in SUBNORMALS] + [F32(-v) for v in SUBNORMALS]
  return np.array(vals, dtype=F32)


def _random_values(rng, n):
  e = rng.integers(-40, 21, n)
  m = rng.uniform(1.0, 2.0, n)
  sgn = np.where(rng.random(n) < 0.5, -1.0, 1.0)
  return (sgn * m * 2.0 ** e).astype(F32)


def _check_split(torch, _lib, lib, a, s, where, aligned_too=False):
  """splits a at scale 2^s, compares every plane byte, sign bit and the K padding with the NumPy restatement,
  the fp16 overflow flag, and the merge (bit for bit, and against the format's bound)"""
  R, C = a.shape
  f16 = _lib.plane_format() == _lib.PLANES_F16
  L = _Layout(f16, R, C)
  src = _dev(torch, a)
  rc, pl = _split(torch, _lib, lib, src, R, C, s)
  _lib.check(rc, "split")
  flag = _lib.plane_overflow()
  with np.errstate(all="ignore"):
    sv = (a * F32(2.0 ** s)).astype(F32)
  raw = _bytes(pl)
  hi, lo, bits = L.planes(raw)
  whi, wlo, wbits = L.want(sv)
  _same_bits(where + " hi", hi, whi)
  _same_bits(where + " lo", lo, wlo)
  assert (hi[:, C:] == 0).all() and (lo[:, C:] == 0).all(), where + ": K padding"
  assert np.array_equal(bits, wbits), where + ": sign bits"
  want_flag = f16 and bool(((np.abs(sv) >= 65520) & np.isfinite(sv)).any())
  assert flag == want_flag, where + ": overflow flag"
  back = _merge(torch, _lib, lib, pl, R, C)
  wm = _merge_np(whi[:, :C], wlo[:, :C], f16)
  assert np.array_equal(np.isnan(back), np.isnan(wm)), where + ": merge NaN"
  ok = ~np.isnan(wm)
  assert np.array_equal(back[ok], wm[ok]), where + ": merge"
  mag = np.abs(sv.astype(np.float64))
  if f16:
    rel = (mag >= 2.0 ** -14) & (mag < 65520)
    tiny = mag < 2.0 ** -14
    _check(where + ": fp16 merge rel", back[rel], sv[rel], 2.0 ** -22 * mag[rel])
    _check(where + ": fp16 merge abs", back[tiny], sv[tiny], 2.0 ** -36)
  else:
    fin = np.isfinite(wm)
    # 2^-22 relative; lo of a value below ~2^-115 is an fp32 subnormal, rounded to a 2^-136 grid
    _check(where + ": tf32 merge", back[fin], sv[fin], 2.0 ** -22 * mag[fin] + 2.0 ** -137)
  if aligned_too and C % 4 == 0:
    # a source 4 bytes off 16-byte alignment takes the scalar loads: same bytes
    buf = torch.zeros(R * C + 4, device="cuda")
    buf[1:1 + R * C] = src.reshape(-1)
    assert (buf.data_ptr() + 4) % 16 != 0
    rc, pl2 = _split(torch, _lib, lib, buf, R, C, s, offset=4)
    _lib.check(rc, "split (unaligned)")
    _lib.plane_overflow()
    assert np.array_equal(_bytes(pl2), raw), where + ": unaligned source"
  return pl


@pytest.mark.parametrize("rows", [1, 7, 8, 9, 33])
@pytest.mark.parametrize("cols", [1, 3, 4, 31, 32, 33, 63, 64, 65, 100, 129])
def test_split_merge_edges(env, rows, cols):
  torch, _lib, lib = env
  rng = np.random.default_rng(rows * 1000 + cols)
  for s in SCALES:
    a = _random_values(rng, rows * cols)
    e = _edge_inputs(s)
    k = min(a.size, e.size)
    a[rng.choice(a.size, k, replace=False)] = rng.permutation(e)[:k]
    _check_split(torch, _lib, lib, a.reshape(rows, cols), s, "%dx%d s=%d" % (rows, cols, s), aligned_too=True)


def test_split_merge_all_edges(env):
  """every edge value at every scale in one tensor, and one tensor of >= 3 grid-stride passes"""
  torch, _lib, lib = env
  rng = np.random.default_rng(5)
  for s in SCALES:
    e = _edge_inputs(s)
    a = _random_values(rng, 8 * 65)
    a[:e.size] = e
    _check_split(torch, _lib, lib, a.reshape(8, 65), s, "all edges s=%d" % s, aligned_too=False)
  for s in (0, -15):
    a = _random_values(rng, 65536 * 100)
    a[rng.choice(a.size, 64, replace=False)] = rng.choice(_edge_inputs(s), 64)
    _check_split(torch, _lib, lib, a.reshape(65536, 100), s, "65536x100 s=%d" % s, aligned_too=True)


def test_split_pins_flt_max(env):
  """FLT_MAX rounds to +Inf in the hi plane (TF32 and fp16 alike), its lo is -Inf, and it merges to NaN; under fp16
  it raises the overflow flag.  The scale is checked at the ABI: +-61 is rejected and writes nothing."""
  torch, _lib, lib = env
  f16 = _lib.plane_format() == _lib.PLANES_F16
  a = np.array([[FLT_MAX, -FLT_MAX, 1.0]], dtype=F32)
  ad = _dev(torch, a)
  rc, pl = _split(torch, _lib, lib, ad, 1, 3)
  _lib.check(rc, "split")
  assert _lib.plane_overflow() == f16
  hi, lo, _ = _Layout(f16, 1, 3).planes(_bytes(pl))
  assert hi[0, 0] == np.inf and lo[0, 0] == -np.inf and hi[0, 1] == -np.inf and lo[0, 1] == np.inf
  assert np.isnan(_merge(torch, _lib, lib, pl, 1, 3)[0, :2]).all()
  for s in (-61, 61):
    rc, pl = _split(torch, _lib, lib, ad, 1, 3, s)
    assert rc == ERR_INVALID
    assert (_bytes(pl) == 0xFF).all()


# ------------------------------------------------------------------------------------------------------------------
# c. the fp32 dense ABI
# ------------------------------------------------------------------------------------------------------------------

def _sms(_lib):
  return _lib.query(_lib.Q_SM_COUNT)


def _dw_splits(B, I, O, sms):
  """dense_simt.cu dw_splits"""
  bn = 16 if O <= 32 else 128
  tiles = -(-I // 128) * -(-O // bn)
  s = -(-2 * sms // tiles)
  return max(1, min(s, -(-B // 256), 64))


def _simt_bwd_ws(B, I, O):
  s = max(1, min(-(-B // 256), 64))
  return -(-((s * I * O + 64 * O) * 4) // 256) * 256


def _colsum_n(rows):
  """rounding chain of simt::colsum: ceil(rps/8) per thread, the 8-term fold, the S2 partials"""
  rps = max(64, -(-(-(-rows // 64)) // 8) * 8)
  s2 = -(-rows // rps)
  return -(-rps // 8) + 8 + s2


def _tc_ok(B, I, O):
  return B >= 128 and I >= 32 and O >= 64


PATHS = ["simt", "auto", "tcgen05"]

# every shape of the former tests/test_gpu_kernels.py test_dense_fwd / test_dense_bwd, and M x N x K over the tile
# tails of both SIMT configurations (BIG 128x128x16, SKINNY 128x16x16 for N <= 32) and the AUTO thresholds
DENSE_SHAPES = sorted(set([
    (256, 100, 64), (1024, 100, 1024), (512, 1024, 1024), (300, 784, 128), (1024, 1024, 10), (7, 5, 3), (129, 33, 17),
    (4096, 512, 512), (128, 100, 10),
    (256, 64, 10), (1024, 1024, 1024), (512, 100, 256), (300, 128, 128), (2048, 1024, 10),
    (1, 1, 1), (1, 17, 33), (127, 15, 16), (127, 1024, 129), (128, 16, 32), (128, 32, 64), (128, 33, 128),
    (129, 17, 1), (129, 100, 33), (129, 1024, 16), (300, 1, 129), (300, 16, 17), (300, 100, 32), (300, 1024, 128),
    (128, 1024, 1), (257, 100, 10), (127, 100, 128),
    (16385, 100, 10), (32768, 256, 64),
]))

_REFS = {}


def _dense_inputs(B, I, O):
  key = (B, I, O)
  if key not in _REFS:
    rng = np.random.default_rng(B * 7919 + I * 31 + O)
    x = rng.standard_normal((B, I)).astype(F32)
    # ReLU mask edges: exact zeros, -0.0 and positive subnormals
    flat = x.reshape(-1)
    n = min(flat.size, 64)
    idx = rng.choice(flat.size, n, replace=False)
    flat[idx[0::3]] = 0.0
    flat[idx[1::3]] = -0.0
    flat[idx[2::3]] = _from_bits(rng.integers(1, 0x800000, idx[2::3].size))
    w = (rng.standard_normal((I, O)) / np.sqrt(I)).astype(F32)
    b = (rng.standard_normal(O) * 0.1).astype(F32)
    dz = (rng.standard_normal((B, O)) / B).astype(F32)
    x64, w64, dz64, b64 = (t.astype(np.float64) for t in (x, w, dz, b))
    ax, aw, adz = np.abs(x64), np.abs(w64), np.abs(dz64)
    y = x64 @ w64
    _REFS.clear()
    _REFS[key] = dict(x=x, w=w, b=b, dz=dz, y=y, yabs=ax @ aw, b64=b64, dw=x64.T @ dz64, dwabs=ax.T @ adz,
                      dx=dz64 @ w64.T, dxabs=adz @ aw.T, db=dz64.sum(0), dbabs=adz.sum(0))
  return _REFS[key]


def _run_dense(torch, _lib, lib, d, B, I, O, act, fws_bytes, bws_bytes):
  sp = _sp(torch)
  xd, wd, bd, dzd = (_dev(torch, d[k]) for k in ("x", "w", "b", "dz"))
  out = {}
  fws = torch.full((max(fws_bytes, 16),), 0xFF, dtype=torch.uint8, device="cuda")
  y = _nan(torch, B, O)
  rc = lib.adn_dense_fwd(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), y.data_ptr(), B, I, O, act, fws.data_ptr(), fws_bytes, sp)
  out["fwd_rc"], out["y"] = rc, y
  y0 = _nan(torch, B, O)
  lib.adn_dense_fwd(xd.data_ptr(), wd.data_ptr(), None, y0.data_ptr(), B, I, O, 0, fws.data_ptr(), fws_bytes, sp)
  out["y0"] = y0
  ws = torch.full((max(bws_bytes, 16) // 4,), float("nan"), device="cuda")
  dx, dw, db = _nan(torch, B, I), _nan(torch, I, O), _nan(torch, O)
  rc = lib.adn_dense_bwd(xd.data_ptr(), wd.data_ptr(), dzd.data_ptr(), dx.data_ptr(), dw.data_ptr(), db.data_ptr(), B, I, O,
                         act, ws.data_ptr(), bws_bytes, sp)
  out["bwd_rc"], out["dx"], out["dw"], out["db"] = rc, dx, dw, db
  dw2 = _nan(torch, I, O)
  lib.adn_dense_bwd(xd.data_ptr(), None, dzd.data_ptr(), None, dw2.data_ptr(), None, B, I, O, act, ws.data_ptr(), bws_bytes, sp)
  out["dw_only"] = dw2
  torch.cuda.synchronize()
  return out


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("B,I,O", DENSE_SHAPES)
def test_dense(gpu, path, B, I, O):
  torch, _lib, lib = gpu
  _lib.set_dense_path({"simt": _lib.PATH_SIMT, "auto": _lib.PATH_AUTO, "tcgen05": _lib.PATH_TCGEN05}[path])
  try:
    d = _dense_inputs(B, I, O)
    tc = path != "simt" and _tc_ok(B, I, O)
    assert _lib.query(_lib.Q_DENSE_FWD_PATH, B, I, O) == (_lib.PATH_TCGEN05 if tc else
                                                         (-1 if path == "tcgen05" else _lib.PATH_SIMT))
    fws_bytes = _lib.query(_lib.Q_DENSE_FWD_WS, B, I, O)
    assert (fws_bytes == 0) == (not tc)
    bws_bytes = _lib.query(_lib.Q_DENSE_BWD_WS, B, I, O)
    assert bws_bytes >= _simt_bwd_ws(B, I, O)
    for act in (0, 1):
      r = _run_dense(torch, _lib, lib, d, B, I, O, act, fws_bytes, bws_bytes)
      if path == "tcgen05" and not tc:
        # forced tensor path on a shape it does not take: an error, and nothing written
        assert r["fwd_rc"] == ERR_UNSUPPORTED and r["bwd_rc"] == ERR_UNSUPPORTED
        for k in ("y", "y0", "dx", "dw", "db", "dw_only"):
          assert torch.isnan(r[k]).all(), k
        return
      _lib.check(r["fwd_rc"], "adn_dense_fwd")
      _lib.check(r["bwd_rc"], "adn_dense_bwd")
      where = "%s %dx%dx%d act%d" % (path, B, I, O, act)
      y = d["y"] + d["b64"]
      if tc:
        yb = TOL * (d["yabs"] + np.abs(d["b64"]))
        y0b = TOL * d["yabs"]
        dxb = TOL * d["dxabs"]
        dwb = TOL * d["dwabs"]
      else:
        yb = _gbound(I + 1, d["yabs"] + np.abs(d["b64"]))           # K FMAs, then the bias add
        y0b = _gbound(I, d["yabs"])
        dxb = _gbound(O, d["dxabs"])                                 # K = out FMAs
        S = _dw_splits(B, I, O, _sms(_lib))
        kps = -(-(-(-B // S)) // 16) * 16
        dwb = _gbound(kps + S, d["dwabs"])                           # k_per_split FMAs, then the S partials in order
      if act:
        y = np.maximum(y, 0)
      _check(where + ": fwd " + ("tc" if tc else "simt"), r["y"].cpu().numpy(), y, yb)
      _check(where + ": fwd nobias " + ("tc" if tc else "simt"), r["y0"].cpu().numpy(), d["y"], y0b)
      keep = d["x"] > 0 if act else np.ones((B, I), dtype=bool)
      dx = r["dx"].cpu().numpy()
      if act:
        assert (dx[~keep] == 0).all(), where + ": dX not masked where x <= 0"
      _check(where + ": dx " + ("tc" if tc else "simt"), dx, d["dx"] * keep, dxb * keep)
      _check(where + ": dw " + ("tc" if tc else "simt"), r["dw"].cpu().numpy(), d["dw"], dwb)
      _check(where + ": db", r["db"].cpu().numpy(), d["db"], _gbound(_colsum_n(B), d["dbabs"]))
      # a repeated call (and the dW-only call) is byte-identical
      r2 = _run_dense(torch, _lib, lib, d, B, I, O, act, fws_bytes, bws_bytes)
      for k in ("y", "y0", "dx", "dw", "db"):
        assert np.array_equal(_bytes(r[k]), _bytes(r2[k])), where + ": repeat " + k
      assert np.array_equal(_bytes(r["dw"]), _bytes(r["dw_only"])), where + ": dW-only call"
      if tc and act:
        # the tensor path always splits into TF32 planes: the process plane format does not change its bytes
        before = _lib.plane_format()
        _lib.set_plane_format(_lib.PLANES_TF32 if before == _lib.PLANES_F16 else _lib.PLANES_F16)
        try:
          r3 = _run_dense(torch, _lib, lib, d, B, I, O, act, fws_bytes, bws_bytes)
        finally:
          _lib.set_plane_format(before)
        for k in ("y", "y0", "dx", "dw", "db"):
          assert np.array_equal(_bytes(r[k]), _bytes(r3[k])), where + ": plane format changed " + k
  finally:
    _lib.set_dense_path(_lib.PATH_AUTO)


def test_dense_path_choice(gpu):
  """AUTO takes the tensor path iff batch >= 128, in >= 32 and out >= 64; SIMT always SIMT; TCGEN05 the tensor path
  or -1.  The forward workspace is 0 exactly when the tensor path is not picked."""
  torch, _lib, lib = gpu
  shapes = [(128, 32, 64)]
  for i in range(3):
    for dlt in (-1, 1):
      s = [128, 32, 64]
      s[i] += dlt
      shapes.append(tuple(s))
  try:
    for path in (_lib.PATH_AUTO, _lib.PATH_SIMT, _lib.PATH_TCGEN05):
      _lib.set_dense_path(path)
      for B, I, O in shapes:
        ok = _tc_ok(B, I, O)
        want = _lib.PATH_SIMT if path == _lib.PATH_SIMT else (_lib.PATH_TCGEN05 if ok else
                                                             (-1 if path == _lib.PATH_TCGEN05 else _lib.PATH_SIMT))
        assert _lib.query(_lib.Q_DENSE_FWD_PATH, B, I, O) == want, (path, B, I, O)
        assert _lib.query(_lib.Q_DENSE_BWD_PATH, B, I, O) == want, (path, B, I, O)
        assert (_lib.query(_lib.Q_DENSE_FWD_WS, B, I, O) == 0) == (want != _lib.PATH_TCGEN05), (path, B, I, O)
  finally:
    _lib.set_dense_path(_lib.PATH_AUTO)


@pytest.mark.parametrize("path", ["simt", "tcgen05"])
def test_dense_workspace_short(gpu, path):
  """a workspace one byte short is ADN_ERR_WORKSPACE and writes nothing; the exact size runs"""
  torch, _lib, lib = gpu
  B, I, O = 300, 100, 70
  _lib.set_dense_path(_lib.PATH_SIMT if path == "simt" else _lib.PATH_TCGEN05)
  try:
    d = _dense_inputs(B, I, O)
    need_b = _simt_bwd_ws(B, I, O) if path == "simt" else _lib.query(_lib.Q_DENSE_BWD_WS, B, I, O)
    need_f = _lib.query(_lib.Q_DENSE_FWD_WS, B, I, O)
    if path == "tcgen05":
      r = _run_dense(torch, _lib, lib, d, B, I, O, 1, need_f - 1, need_b)
      assert r["fwd_rc"] == ERR_WORKSPACE
      assert torch.isnan(r["y"]).all() and torch.isnan(r["y0"]).all()
      _lib.check(r["bwd_rc"], "adn_dense_bwd")
    r = _run_dense(torch, _lib, lib, d, B, I, O, 1, need_f, need_b - 1)
    _lib.check(r["fwd_rc"], "adn_dense_fwd")
    assert r["bwd_rc"] == ERR_WORKSPACE
    for k in ("dx", "dw", "db", "dw_only"):
      assert torch.isnan(r[k]).all(), k
    r = _run_dense(torch, _lib, lib, d, B, I, O, 1, need_f, need_b)
    _lib.check(r["bwd_rc"], "adn_dense_bwd")
  finally:
    _lib.set_dense_path(_lib.PATH_AUTO)


# ------------------------------------------------------------------------------------------------------------------
# d. adn_colsum
# ------------------------------------------------------------------------------------------------------------------

COLSUM_SHAPES = [(r, c) for r in (1, 63, 64, 65, 4095, 4096, 4097, 65537) for c in (1, 31, 32, 33, 1000)] + [(5000, 10)]


@pytest.mark.parametrize("rows,cols", COLSUM_SHAPES)
def test_colsum(gpu, rows, cols):
  torch, _lib, lib = gpu
  rng = np.random.default_rng(rows * 7 + cols)
  x = rng.standard_normal((rows, cols), dtype=F32)
  xd = _dev(torch, x)
  nb = _lib.query(_lib.Q_COLSUM_WS, rows, cols)
  assert nb >= 64 * cols * 4
  outs = []
  for _ in range(2):
    ws = torch.full((nb // 4,), float("nan"), device="cuda")
    out = _nan(torch, cols)
    _lib.check(lib.adn_colsum(xd.data_ptr(), rows, cols, out.data_ptr(), ws.data_ptr(), nb, _sp(torch)), "adn_colsum")
    outs.append(out)
  ref = x.sum(axis=0, dtype=np.float64)
  bound = _gbound(_colsum_n(rows), np.abs(x).sum(axis=0, dtype=np.float64))
  _check("%dx%d: colsum" % (rows, cols), outs[0].cpu().numpy(), ref, bound)
  assert np.array_equal(_bytes(outs[0]), _bytes(outs[1])), "repeat"
  out = _nan(torch, cols)
  ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")
  assert lib.adn_colsum(xd.data_ptr(), rows, cols, out.data_ptr(), ws.data_ptr(), 64 * cols * 4 - 1, _sp(torch)) == ERR_WORKSPACE
  assert torch.isnan(out).all()
