"""GPU tests of the grouped launches of a training step other than the plane GEMM waves, in BOTH plane formats:
adn_head_group (every subnetwork loss and ensemble head), adn_opt_step_group (every optimizer, with the weight-plane
refresh), adn_head_bookkeeping (EMA + loss trace) and the MATRIX-mixture helpers adn_l1_norm / adn_l1_grad_add.

Every output is compared element by element with a float64 NumPy restatement of the same operation.  Where a kernel
consumes an earlier stage's output, the reference is evaluated on the kernel's own fp32 output of that stage (the
gradient from the kernel's ensemble logits, the optimizer update from the state before the step), so errors do not
compound.  Each bound is componentwise, gamma(n) * sum|terms| with gamma(n) = n u / (1 - n u) and u = 2^-24, where
n is the longest chain of roundings an element goes through in the kernel's summation order (written out beside each
bound).  A bound relative to a global maximum could not see a wrong small entry.

A grouped call that rejects one of its ops must not have changed anything: the last tests make the last op of a call
that spans several launches invalid and check every output, parameter, slot, plane and step counter afterwards.
"""

import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F32 = np.float32
ERR_INVALID, ERR_UNSUPPORTED, ERR_WORKSPACE = -22, -95, -12

_WORST = {}    # check name -> largest |err| / bound seen in this module (printed at teardown, pytest -s)


def _gamma(n):
  return n * U / (1.0 - n * U)


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
  _lib.set_plane_format(_lib.PLANES_F16 if request.param == "f16" else _lib.PLANES_TF32)
  _lib.plane_overflow()      # clear the sticky flag
  yield torch, _lib, lib
  _lib.set_plane_format(before)


def _sp(torch):
  return torch.cuda.current_stream().cuda_stream


def _dev(torch, a):
  return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _np(t):
  return t.cpu().numpy()


def _bytes(t):
  import torch
  return t.reshape(-1).view(torch.uint8).cpu().numpy()


def _ptr(t):
  return None if t is None else t.data_ptr()


def _plane_regions(f16, rows, cols):
  """byte ranges of the hi and lo planes' [nkb][rows][BK] regions in a plane buffer"""
  bk, es = (64, 2) if f16 else (32, 4)
  n = -(-cols // bk) * rows * bk
  elems = -(-n // 128) * 128
  return slice(0, n * es), slice(elems * es, elems * es + n * es)


def _split(torch, _lib, lib, src, rows, cols, log2_scale=0):
  """adn_planes_split_scaled of a device tensor into a fresh zeroed buffer (uint8)"""
  out = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, rows, cols),), dtype=torch.uint8, device="cuda")
  _lib.check(lib.adn_planes_split_scaled(src.data_ptr(), rows, cols, out.data_ptr(), log2_scale, _sp(torch)), "split")
  return out


# ------------------------------------------------------------------------------------------------------------------
# heads
# ------------------------------------------------------------------------------------------------------------------

ROWS = 128      # examples per CTA of the head kernel


def _n_max(C):
  """largest n_members whose shared-memory tile fits 227 KiB (csrc/heads.cu head_smem_bytes)"""
  n = 1
  while n < 64 and ((n + 2) * ROWS * C + 4 * max(C, n + 1)) * 4 <= 227 * 1024:
    n += 1
  return n


def _fin_depth(B):
  """additions along the longest chain of the finalize over the per-CTA partials: lanes stride over n_cta partials
  then a 5-level shuffle tree; above 512 CTAs a first level (256 threads strided + 5 shuffles + 8 warps) and then
  the single-row finalize (1 + 5)"""
  n_cta = -(-B // ROWS)
  if n_cta > 512:
    return -(-n_cta // 256) + 5 + 8 + 1 + 5
  return -(-n_cta // 32) + 5


class _Head:
  """One head op: numpy inputs, device tensors, and which outputs the group call asks for."""

  def __init__(self, **kw):
    self.__dict__.update(kw)


def _head_inputs(torch, B, C, seed):
  rng = np.random.default_rng(seed)
  P = _n_max(C)
  pool = [(rng.standard_normal((B, C)) * 2.0).astype(F32) for _ in range(P)]
  labels = rng.integers(0, C, size=B).astype(np.int64)
  lab_mse = rng.standard_normal((B, C)).astype(F32)
  lab_sig = rng.uniform(0.0, 1.0, (B, C)).astype(F32)
  lab_sig[::3] = np.round(lab_sig[::3])
  d = dict(pool=pool, pool_d=[_dev(torch, m) for m in pool], labels=labels, lab_mse=lab_mse, lab_sig=lab_sig)
  d.update(labels_d=_dev(torch, labels), lab_mse_d=_dev(torch, lab_mse), lab_sig_d=_dev(torch, lab_sig))
  return d, rng


def _labels_of(inp, head):
  if head == 0:
    return inp["labels_d"], None
  return None, (inp["lab_mse_d"] if head == 1 else inp["lab_sig_d"])


def _make_head_ops(torch, _lib, inp, rng, B, C, n_ops):
  """A mixed group: every third op a colsum-only sub-loss op (dlogits dense / as scaled planes, logits-layer db), the
  others SCALAR / VECTOR ensemble heads of all three kinds with 1..n_max members, with and without bias, w, dw, dbias,
  dens and ens_out, reg_multiplier 1 and 2, reg_is_zero set and clear."""
  P = len(inp["pool"])
  nan = float("nan")
  ops = []
  nc = ne = 0
  for i in range(n_ops):
    if i % 3 == 0:
      c = nc
      nc += 1
      head = c % 3
      k = i % P
      o = _Head(head=head, mix=_lib.MIX_SCALAR, colsum=True, members=[k], w=None, bias=None,
                gammas=np.zeros(1, F32), reg_is_zero=1, reg_mult=1.0, scale=[30, 0, 15, 7][c % 4],
                want_dens=c % 2 == 0, want_planes=c % 4 != 2, want_dbias=c % 3 != 2, want_dw=False, want_ens=False)
    else:
      j = ne
      ne += 1
      head = j % 3
      mix = _lib.MIX_SCALAR if (j // 3) % 2 == 0 else _lib.MIX_VECTOR
      N = [1, P, 2, min(3, P), max(1, P // 2), P][j % 6]
      members = [(i + k) % P for k in range(N)]
      wshape = (N,) if mix == _lib.MIX_SCALAR else (N, C)
      if j % 5 == 4:
        w = None
      else:
        w = rng.standard_normal(wshape).astype(F32)
        w.reshape(-1)[0] = 0.0                  # sign(0) = 0: no regulariser gradient
      o = _Head(head=head, mix=mix, colsum=False, members=members, w=w,
                bias=rng.standard_normal(C).astype(F32) if j % 2 == 0 else None,
                gammas=rng.uniform(0.01, 0.2, N).astype(F32), reg_is_zero=int(j % 7 == 6),
                reg_mult=2.0 if j % 2 else 1.0, scale=0, want_dens=j % 2 == 1, want_planes=False,
                want_dbias=j % 3 != 1, want_dw=j % 4 != 3, want_ens=j % 3 != 2)
    o.N = len(o.members)
    o.w_d = None if o.w is None else _dev(torch, o.w)
    o.bias_d = None if o.bias is None else _dev(torch, o.bias)
    o.lab, o.labf = _labels_of(inp, o.head)
    o.ws_bytes = _lib.query(_lib.Q_HEAD_WS, B, C, o.N)
    o.ws = torch.empty((o.ws_bytes,), dtype=torch.uint8, device="cuda")
    o.out3 = torch.full((3,), nan, device="cuda")
    o.dens = torch.full((B, C), nan, device="cuda") if o.want_dens else None
    o.ens = torch.full((B, C), nan, device="cuda") if o.want_ens else None
    o.dbias = torch.full((C,), nan, device="cuda") if o.want_dbias else None
    wsz = 0 if o.colsum else (o.N if o.mix == _lib.MIX_SCALAR else o.N * C)
    o.dw = torch.full((wsz,), nan, device="cuda") if o.want_dw else None
    o.planes = (torch.full((_lib.query(_lib.Q_PLANES_BYTES, B, C),), 255, dtype=torch.uint8, device="cuda")
                if o.want_planes else None)
    o.members_host = _lib.ptr_array([inp["pool_d"][k].data_ptr() for k in o.members])
    o.gammas_host = _lib.f32_array(o.gammas)
    ops.append(o)
  return ops


def _head_struct(_lib, o):
  return _lib.HeadOp(o.head, o.mix, ctypes.cast(o.members_host, ctypes.POINTER(ctypes.c_void_p)), o.N, o.reg_is_zero,
                     _ptr(o.w_d), _ptr(o.bias_d), ctypes.cast(o.gammas_host, ctypes.POINTER(ctypes.c_float)),
                     o.reg_mult, o.scale, _ptr(o.lab), _ptr(o.labf), o.out3.data_ptr(), _ptr(o.dw), _ptr(o.dbias),
                     _ptr(o.dens), _ptr(o.ens), _ptr(o.planes), int(o.colsum), 0, o.ws.data_ptr(), o.ws_bytes)


def _run_alone(torch, _lib, lib, o, B, C):
  """The same op through adn_head_loss_p / adn_ensemble_head, always with dens and ens_out (and planes and column
  sums for a sub-loss op).  Returns numpy outputs."""
  nan = float("nan")
  sp = _sp(torch)
  ws = torch.empty((o.ws_bytes,), dtype=torch.uint8, device="cuda")
  dens = torch.full((B, C), nan, device="cuda")
  dbias = torch.full((C,), nan, device="cuda")
  r = {}
  if o.colsum:
    loss = torch.full((1,), nan, device="cuda")
    planes = torch.full((_lib.query(_lib.Q_PLANES_BYTES, B, C),), 255, dtype=torch.uint8, device="cuda")
    _lib.check(lib.adn_head_loss_p(o.head, o.members_host[0], _ptr(o.lab), _ptr(o.labf), loss.data_ptr(),
                                   dens.data_ptr(), planes.data_ptr(), dbias.data_ptr(), o.scale, B, C, ws.data_ptr(),
                                   o.ws_bytes, sp), "adn_head_loss_p")
    r.update(loss=_np(loss), planes=_bytes(planes), planes_d=planes)
  else:
    out3 = torch.full((3,), nan, device="cuda")
    ens = torch.full((B, C), nan, device="cuda")
    dw = torch.full((o.dw.numel(),), nan, device="cuda") if o.dw is not None else None
    _lib.check(lib.adn_ensemble_head(o.head, o.mix, o.members_host, o.N, _ptr(o.w_d), _ptr(o.bias_d), o.gammas_host,
                                     o.reg_is_zero, o.reg_mult, _ptr(o.lab), _ptr(o.labf), out3.data_ptr(), _ptr(dw),
                                     dbias.data_ptr(), dens.data_ptr(), ens.data_ptr(), B, C, ws.data_ptr(), o.ws_bytes, sp),
               "adn_ensemble_head")
    r.update(out3=_np(out3), ens=_np(ens), dw=None if dw is None else _np(dw))
  r.update(dens=_np(dens), dens_d=dens, dbias=_np(dbias))
  return r


def _check_loss_and_grad(tag, head, e, lab, labf, B, C, dens, loss):
  """loss = out3[0] and dens = dLoss/d ens, evaluated on the kernel's ensemble logits e [B, C] (float64)"""
  D = 9 + _fin_depth(B)              # per-CTA block tree (5 shuffles + 4 warps), then the finalize
  if head == 0:
    # ex_c = expf(fl(e_c - mx)): rel (|z_c| + 4) u (argument rounding, expf <= 2 ulp); s: C - 1 sequential adds;
    # p_c = ex_c * fl(1/s): rel <= (C + 9 + 2M) u with M = max |z|; fl(fl(p - onehot) * fl(1/B)): 3 u |p - onehot|
    mx = e.max(axis=1, keepdims=True)
    z = e - mx
    ex = np.exp(z)
    s = ex.sum(axis=1, keepdims=True)
    p = ex / s
    onehot = np.zeros_like(e)
    onehot[np.arange(B), lab] = 1.0
    g = (p - onehot) / B
    M = np.abs(z).max(axis=1, keepdims=True)
    _check(tag + ": dens softmax", dens, g, 1.0001 * U * ((C + 10 + 2 * M) * p + 3 * np.abs(p - onehot)) / B)
    zy = z[np.arange(B), lab]
    lr = np.log(s[:, 0]) - zy
    # loss_r = -(zy - logf(s)): |zy| u + (C + 3 + M) u (s) + 2 u |log s| (logf) + u |loss_r|
    t_r = np.abs(zy) + C + 3 + M[:, 0] + 2 * np.abs(np.log(s[:, 0])) + np.abs(lr)
    want = lr.sum() / B
    _check(tag + ": loss softmax", loss, want, 1.0001 * (U * t_r.sum() + _gamma(D) * np.abs(lr).sum()) / B
           + U * abs(want))
  elif head == 1:
    d = e - labf
    g = 2.0 * d / (B * C)
    # fl(e - y), fl(2 d * fl(1/(B C))): three roundings
    _check(tag + ": dens mse", dens, g, _gamma(3) * np.abs(g))
    # loss_r = sum_c fl(d^2), d^2 carries 3 u, C sequential adds; the batch tree; / (B C)
    lr = (d * d).sum(axis=1)
    want = lr.sum() / (B * C)
    _check(tag + ": loss mse", loss, want, _gamma(C + 3 + D) * lr.sum() / (B * C) + U * want)
  else:
    E = np.exp(-np.abs(e))
    sig = 1.0 / (1.0 + np.exp(-e))
    g = (sig - labf) / (B * C)
    # expf(-x) <= 4 u, 1 + E, 1 / (..): sig rel 6 u; fl(sig - z) and * fl(1/(B C)): 3 u |sig - z|
    _check(tag + ": dens sigmoid", dens, g, 1.0001 * U * (6 * sig + 3 * np.abs(sig - labf)) / (B * C))
    a, xz, lp = np.maximum(e, 0), e * labf, np.log1p(E)
    lr = (a - xz + lp).sum(axis=1)
    # per element: fl(x z), log1pf(expf) (6 u lp), two adds; per row C sequential adds; then the batch tree
    tau = (a + np.abs(xz) + lp).sum(axis=1)
    want = lr.sum() / (B * C)
    _check(tag + ": loss sigmoid", loss, want, (_gamma(C + 8) * tau.sum() + _gamma(D) * np.abs(lr).sum()) / (B * C)
           + U * abs(want))


def _check_head(tag, o, inp, r, B, C, _lib):
  """every output of the op run alone against its float64 restatement"""
  pool = inp["pool"]
  mem = [pool[k].astype(np.float64) for k in o.members]
  lab, labf = inp["labels"], (inp["lab_mse"] if o.head == 1 else inp["lab_sig"]).astype(np.float64)
  if o.colsum:
    e = mem[0]           # weight 1, no bias: the ensemble logits are the logits themselves
    loss = r["loss"][0]
  else:
    mix = o.mix
    if o.w is None:
      wk = [np.ones(1 if mix == _lib.MIX_SCALAR else C)] * o.N
    elif mix == _lib.MIX_SCALAR:
      wk = [np.full(1, o.w[k], np.float64) for k in range(o.N)]
    elif mix == _lib.MIX_VECTOR:
      wk = [o.w[k].astype(np.float64) for k in range(o.N)]
    else:
      wk = [np.ones(C)] * o.N
    b = np.zeros(C) if o.bias is None else o.bias.astype(np.float64)
    terms = [wk[k] * mem[k] for k in range(o.N)]
    ref = b + sum(terms)
    # v = bias; v += w_k m_k for k = 0..N-1: N additions and one product rounding per term
    _check(tag + ": ens_out", r["ens"], ref, _gamma(o.N + 1) * (np.abs(b) + sum(np.abs(t) for t in terms)))
    e = r["ens"].astype(np.float64)
    loss = r["out3"][0]
  dens = r["dens"].astype(np.float64)
  _check_loss_and_grad(tag, o.head, e, lab, labf, B, C, dens, loss)
  fin = _fin_depth(B)
  # thread (warp w, column c): 32 rows in sequence, then the 4 warps, then the finalize
  _check(tag + ": dbias", r["dbias"], dens.sum(axis=0), _gamma(36 + fin) * np.abs(dens).sum(axis=0))
  if o.colsum:
    return
  out3 = r["out3"].astype(np.float64)
  wdim = 1 if o.mix == _lib.MIX_SCALAR else C
  if o.reg_is_zero:
    assert out3[1] == 0.0
  else:
    if o.mix == _lib.MIX_MATRIX:
      l1 = o.w.astype(np.float64)
    elif o.w is None:
      l1 = np.full(o.N, float(wdim))
    else:
      l1 = np.abs(o.w.astype(np.float64).reshape(o.N, wdim)).sum(axis=1)
    g64 = o.gammas.astype(np.float64)
    # l1_k: wdim sequential adds; reg = sum_k fl(gamma_k l1_k) in sequence
    _check(tag + ": reg", out3[1], (g64 * l1).sum(), _gamma(wdim + o.N + 1) * (g64 * l1).sum())
  assert r["out3"][2] == F32(r["out3"][0] + r["out3"][1])
  if r.get("dw") is None:
    return
  dw = r["dw"].astype(np.float64).reshape(o.N, wdim)
  if o.w is None:
    sgn = np.ones((o.N, wdim))
  else:
    sgn = np.sign(o.w.astype(np.float64).reshape(o.N, wdim))
  reg = (0.0 if o.reg_is_zero else 1.0) * (F32(o.reg_mult) * o.gammas).astype(np.float64)[:, None] * sgn
  for k in range(o.N):
    prod = dens * mem[k]
    if o.mix == _lib.MIX_SCALAR:
      # row dot product (C fused adds), 5 shuffles + 4 warps, the finalize, + the regulariser term
      t, tb = prod.sum(), np.abs(prod).sum()
      n = C + 11 + fin
    else:
      # one product, 5 shuffles + 4 warps, the finalize, + the regulariser term
      t, tb = prod.sum(axis=0), np.abs(prod).sum(axis=0)
      n = 11 + fin
    _check(tag + ": dw", dw[k], t + reg[k], _gamma(n) * tb + 2 * U * np.abs(reg[k]))


HEAD_SHAPES = [(1, 1, 9), (127, 2, 9), (128, 3, 9), (129, 4, 9), (1000, 10, 30), (32768, 16, 9), (65536, 5, 9),
               (65537, 17, 26), (129, 64, 9)]


@pytest.mark.parametrize("B,C,n_ops", HEAD_SHAPES)
def test_head_group(env, B, C, n_ops):
  """adn_head_group: every output against float64, the gradient planes byte-identical to adn_planes_split_scaled of
  the kernel's own dlogits (zero padding columns included), the fp16 overflow flag, and every op byte-identical to
  the same op run alone.  30 and 26 ops take two launches; batch 65537 (> 512 CTAs) runs op by op with the two-level
  finalize."""
  torch, _lib, lib = env
  f16 = _lib.plane_format() == _lib.PLANES_F16
  inp, rng = _head_inputs(torch, B, C, B * 100 + C)
  ops = _make_head_ops(torch, _lib, inp, rng, B, C, n_ops)
  arr = (_lib.HeadOp * n_ops)(*[_head_struct(_lib, o) for o in ops])
  _lib.plane_overflow()
  _lib.check(lib.adn_head_group(arr, n_ops, B, C, _sp(torch)), "adn_head_group")
  got_ovf = _lib.plane_overflow()
  want_ovf = False
  hi_r, lo_r = _plane_regions(f16, B, C)
  for i, o in enumerate(ops):
    tag = "op %d" % i
    r = _run_alone(torch, _lib, lib, o, B, C)
    # byte-identical to the op alone
    if o.colsum:
      out3 = _np(o.out3)
      assert out3[0].tobytes() == r["loss"][0].tobytes(), tag
      assert out3[1] == 0.0 and out3[2].tobytes() == out3[0].tobytes(), tag
    else:
      assert _np(o.out3).tobytes() == r["out3"].tobytes(), tag
      if o.ens is not None:
        assert _np(o.ens).tobytes() == r["ens"].tobytes(), tag
      if o.dw is not None:
        assert _np(o.dw).tobytes() == r["dw"].tobytes(), tag
    if o.dens is not None:
      assert _np(o.dens).tobytes() == r["dens"].tobytes(), tag
    if o.dbias is not None:
      assert _np(o.dbias).tobytes() == r["dbias"].tobytes(), tag
    if o.planes is not None:
      gp = _bytes(o.planes)
      assert gp.tobytes() == r["planes"].tobytes(), tag
      ref = _bytes(_split(torch, _lib, lib, r["dens_d"], B, C, o.scale))
      assert (gp[hi_r] == ref[hi_r]).all() and (gp[lo_r] == ref[lo_r]).all(), tag + ": planes"
      v = np.abs(r["dens"].astype(np.float64) * 2.0 ** o.scale)
      want_ovf |= bool(((v >= 65520.0) & np.isfinite(v)).any())
    _check_head(tag, o, inp, r, B, C, _lib)
  assert got_ovf == (want_ovf and f16)
  if B <= 1000 and C > 1:
    assert want_ovf          # op 0 carries dlogits * 2^30: the overflow case is exercised
  _lib.plane_overflow()


@pytest.mark.parametrize("head", [0, 1, 2])
@pytest.mark.parametrize("B,C", [(1000, 5), (129, 33), (300, 10)])
def test_matrix_mixture(env, head, B, C):
  """MATRIX mixture: members arrive multiplied by their matrices, w = their L1 norms from adn_l1_norm, dw must be
  NULL (and is rejected otherwise, alone and in a group)."""
  torch, _lib, lib = env
  inp, rng = _head_inputs(torch, B, C, 7 * B + C + head)
  N = min(3, len(inp["pool"]))
  Ws = [rng.standard_normal((17, C)).astype(F32) for _ in range(N)]
  l1 = torch.full((N,), float("nan"), device="cuda")
  for k in range(N):
    _lib.check(lib.adn_l1_norm(_dev(torch, Ws[k]).data_ptr(), Ws[k].size, l1.data_ptr() + 4 * k, _sp(torch)), "l1")
  torch.cuda.synchronize()
  o = _Head(head=head, mix=_lib.MIX_MATRIX, colsum=False, members=list(range(N)), N=N, w=_np(l1),
            bias=rng.standard_normal(C).astype(F32), gammas=rng.uniform(0.01, 0.2, N).astype(F32), reg_is_zero=0,
            reg_mult=2.0, scale=0, want_planes=False)
  o.w_d, o.bias_d = l1, _dev(torch, o.bias)
  o.lab, o.labf = _labels_of(inp, head)
  o.ws_bytes = _lib.query(_lib.Q_HEAD_WS, B, C, N)
  o.ws = torch.empty((o.ws_bytes,), dtype=torch.uint8, device="cuda")
  o.members_host = _lib.ptr_array([inp["pool_d"][k].data_ptr() for k in o.members])
  o.gammas_host = _lib.f32_array(o.gammas)
  o.dw, o.dbias = None, torch.empty((C,), device="cuda")
  r = _run_alone(torch, _lib, lib, o, B, C)
  _check_head("matrix", o, inp, r, B, C, _lib)
  # reg = sum_k gamma_k * ||W_k||_1 against the matrices themselves (adn_l1_norm: 1 element per thread, 10 levels)
  want = sum(float(o.gammas[k]) * np.abs(Ws[k].astype(np.float64)).sum() for k in range(N))
  _check("matrix reg vs W", r["out3"][1], want, _gamma(10 + N + 2) * want)
  dw = torch.empty((N,), device="cuda")
  rc = lib.adn_ensemble_head(head, _lib.MIX_MATRIX, o.members_host, N, l1.data_ptr(), None, o.gammas_host, 0, 1.0,
                             _ptr(o.lab), _ptr(o.labf), torch.empty(3, device="cuda").data_ptr(), dw.data_ptr(), None,
                             None, None, B, C, o.ws.data_ptr(), o.ws_bytes, _sp(torch))
  assert rc == ERR_INVALID and "dw must be NULL" in lib.adn_last_error().decode()
  o.out3, o.dens, o.ens, o.planes, o.dw = torch.empty(3, device="cuda"), None, None, None, dw
  op = _head_struct(_lib, o)
  assert lib.adn_head_group((_lib.HeadOp * 1)(op), 1, B, C, _sp(torch)) == ERR_INVALID
  assert "op 0: dw must be NULL" in lib.adn_last_error().decode()


@pytest.mark.parametrize("head", [0, 1, 2])
@pytest.mark.parametrize("mix", [0, 1])
@pytest.mark.parametrize("C", [4, 5, 17, 33, 64])
def test_unaligned_member(env, head, mix, C):
  """A member 4 bytes off 16-byte alignment takes the __ldg path instead of cp.async: same outputs, byte for byte."""
  torch, _lib, lib = env
  B = 300
  inp, rng = _head_inputs(torch, B, C, 11 * C + head + mix)
  N = min(3, len(inp["pool"]))
  raw = torch.empty((B * C + 1,), device="cuda")
  raw[1:].copy_(inp["pool_d"][1].view(-1))
  view = raw[1:]
  assert view.data_ptr() % 16 == 4
  w = rng.standard_normal((N,) if mix == 0 else (N, C)).astype(F32)
  w_d, b_d = _dev(torch, w), _dev(torch, rng.standard_normal(C).astype(F32))
  gam = _lib.f32_array(rng.uniform(0.01, 0.2, N))
  lab, labf = _labels_of(inp, head)
  ws_bytes = _lib.query(_lib.Q_HEAD_WS, B, C, N)
  outs = []
  for m1 in (inp["pool_d"][1], view):
    o = [torch.full(s, float("nan"), device="cuda") for s in ((3,), w.shape, (C,), (B, C), (B, C))]
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device="cuda")
    members = _lib.ptr_array([inp["pool_d"][0].data_ptr(), m1.data_ptr()] + [p.data_ptr() for p in inp["pool_d"][2:N]])
    _lib.check(lib.adn_ensemble_head(head, mix, members, N, w_d.data_ptr(), b_d.data_ptr(), gam, 0, 2.0, _ptr(lab),
                                     _ptr(labf), *[t.data_ptr() for t in o], B, C, ws.data_ptr(), ws_bytes,
                                     _sp(torch)), "adn_ensemble_head")
    outs.append([_np(t).tobytes() for t in o])
  assert outs[0] == outs[1]


# ------------------------------------------------------------------------------------------------------------------
# bookkeeping and the L1 helpers
# ------------------------------------------------------------------------------------------------------------------

def _book_setup(torch, _lib, n, seed):
  rng = np.random.default_rng(seed)
  caps = [[1, 3, 4][i % 3] for i in range(n)]
  decays = [[0.9, 0.5, 0.99][i % 3] for i in range(n)]
  ema = [torch.zeros(3, device="cuda") for _ in range(n)]
  out3 = [torch.zeros(3, device="cuda") for _ in range(n)]
  sub = [torch.zeros(1, device="cuda") for _ in range(n)]
  trace = [_dev(torch, rng.standard_normal((c, 4)).astype(F32)) for c in caps]
  books = (_lib.HeadBook * n)(*[_lib.HeadBook(ema[i].data_ptr(), out3[i].data_ptr(), sub[i].data_ptr(),
                                              trace[i].data_ptr(), decays[i], caps[i]) for i in range(n)])
  return rng, caps, decays, ema, out3, sub, trace, books


@pytest.mark.parametrize("n", [1, 64, 65, 130])
def test_head_bookkeeping(env, n):
  """Zero-debiased EMA against the float64 recurrence from the kernel's previous state, trace rows exact, capacities
  1, 3 and 4 over more steps than the capacity; the step counter is an int64 past 2^32."""
  torch, _lib, lib = env
  rng, caps, decays, ema, out3, sub, trace, books = _book_setup(torch, _lib, n, n)
  want_trace = [_np(t) for t in trace]
  step_d = torch.zeros((), dtype=torch.int64, device="cuda")
  for step in [0, 1, 2, 3, 4, 5, 6, 2 ** 33 + 5]:
    step_d.fill_(step)
    x = rng.standard_normal((n, 3)).astype(F32)
    s = rng.standard_normal(n).astype(F32)
    for i in range(n):
      out3[i].copy_(torch.as_tensor(x[i]))
      sub[i].fill_(float(s[i]))
    before = [_np(e).astype(np.float64) for e in ema]
    _lib.check(lib.adn_head_bookkeeping(books, n, step_d.data_ptr(), _sp(torch)), "adn_head_bookkeeping")
    for i in range(n):
      got = _np(ema[i])
      b, cnt = before[i][0], before[i][1]
      d = float(F32(decays[i]))
      xb = float(x[i, 2])
      # biased - (biased - x) (1 - decay): three roundings ((1 - decay) is exact)
      nb = b - (b - xb) * (1 - d)
      _check("ema biased", got[0], nb, _gamma(3) * (abs(b) + abs(b - xb) * (1 - d)))
      assert got[1] == cnt + 1
      # fl(biased / fl(1 - powf(decay, n))): powf <= 4 ulp, the subtraction and the division
      P = d ** (cnt + 1)
      v = float(got[0]) / (1 - P)
      _check("ema value", got[2], v, 1.0001 * U * (8 * P / (1 - P) + 2) * abs(v))
      want_trace[i][step % caps[i]] = [s[i], x[i, 0], x[i, 2], got[2]]
      assert np.array_equal(_np(trace[i]), want_trace[i]), (i, step)


@pytest.mark.parametrize("n", [1, 255, 257, 1024 * 256 + 1])
def test_l1_grad_add(env, n):
  """dw += coef * sign(w), exact against np.float32 arithmetic, w with +0 and -0 entries (sign 0)."""
  torch, _lib, lib = env
  rng = np.random.default_rng(n)
  w = rng.standard_normal(n).astype(F32)
  w[::7] = 0.0
  w[3::7] = -0.0
  dw = rng.standard_normal(n).astype(F32)
  dw[5::11] = -0.0
  coef = F32(0.37)
  dw_d = _dev(torch, dw)
  _lib.check(lib.adn_l1_grad_add(dw_d.data_ptr(), _dev(torch, w).data_ptr(), n, coef, _sp(torch)), "l1_grad_add")
  sgn = np.where(w > 0, F32(1), np.where(w < 0, F32(-1), F32(0))).astype(F32)
  want = (dw + coef * sgn).astype(F32)
  assert np.array_equal(_np(dw_d).view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("n", [0, 1, 1025, 10 ** 7])
def test_l1_norm(env, n):
  """sum |x|: each of 1024 threads adds ceil(n/1024) elements in sequence, then a 10-level tree."""
  torch, _lib, lib = env
  rng = np.random.default_rng(n + 1)
  x = rng.standard_normal(max(n, 1)).astype(F32)
  out = torch.full((1,), float("nan"), device="cuda")
  _lib.check(lib.adn_l1_norm(_dev(torch, x).data_ptr(), n, out.data_ptr(), _sp(torch)), "l1_norm")
  a = np.abs(x[:n].astype(np.float64))
  _check("l1_norm", _np(out)[0], a.sum(), _gamma(-(-n // 1024) + 10) * a.sum())
  if n == 0:
    assert _np(out)[0] == 0.0


# ------------------------------------------------------------------------------------------------------------------
# optimizers
# ------------------------------------------------------------------------------------------------------------------

SGD, MOM, RMS, ADAM, COS = 0, 1, 2, 3, 4
HYPER = {SGD: [0.1], MOM: [0.05, 0.9], RMS: [0.01, 0.9, 0.5, 1e-7], ADAM: [0.01, 0.9, 0.999, 1e-7],
         COS: [0.1, 0.9, 2.5, 0.1]}
N_SLOTS = {SGD: 0, MOM: 1, COS: 1, RMS: 2, ADAM: 2}
# shapes of the parameters: hidden and logits kernels, odd shapes, chunk boundaries (4096 elements) inside rows with
# cols % 4 == 0 ([90, 120]) and not ([37, 129], [3, 4097] = 4096 * 3 + 3 elements), biases of 1, 3 and 5000
SHAPES = [(100, 64), (64, 128), (128, 10), (1, 4), (3, 5), (37, 129), (90, 120), (3, 4097), (1,), (3,), (5000,)]
NO_PLANES = {(128, 10), (3, 5)}        # 2-D parameters whose planes_host entry is NULL


class _Opt:
  """One optimizer of a group: its parameters, gradients, slots, weight planes and step counter on the device."""

  def __init__(self, torch, _lib, lib, rng, kind, shapes, step0, offset):
    self.kind, self.shapes, self.offset = kind, shapes, offset
    self.hyper = [float(F32(h)) for h in HYPER[kind]]
    self.step = None if step0 is None else torch.full((), step0, dtype=torch.int64, device="cuda")
    self.p, self.g, self.s0, self.s1, self.planes, self.cols = [], [], [], [], [], []
    self._keep = []
    for sh in shapes:
      n = int(np.prod(sh))
      self.p.append(self._alloc(torch, rng.standard_normal(n)))
      self.g.append(self._alloc(torch, np.zeros(n)))
      # slots: accumulator / mean square (> 0) / first moment, then RMSProp momentum / Adam second moment (> 0)
      s0 = None if kind == SGD else (rng.uniform(0.5, 1.5, n) if kind == RMS else rng.standard_normal(n) * 0.1)
      s1 = {RMS: rng.standard_normal(n) * 0.01, ADAM: rng.uniform(0.01, 0.1, n)}.get(kind)
      self.s0.append(None if s0 is None else self._alloc(torch, s0))
      self.s1.append(None if s1 is None else self._alloc(torch, s1))
      if len(sh) == 2 and sh not in NO_PLANES:
        pl = _split(torch, _lib, lib, self.p[-1], sh[0], sh[1])
        self.planes.append(pl)
        self.cols.append(sh[1])
      else:
        self.planes.append(None)
        self.cols.append(0)
    self.arrays = [_lib.ptr_array([_ptr(t) for t in ts]) for ts in (self.p, self.g, self.s0, self.s1, self.planes)]
    self.sizes = _lib.i64_array([int(np.prod(sh)) for sh in shapes])
    self.cols_h = _lib.i64_array(self.cols)
    self.hyper_h = _lib.f32_array(self.hyper)

  def _alloc(self, torch, a):
    """a device fp32 tensor holding `a`; with offset, a view 4 bytes past a 16-byte boundary"""
    a = np.asarray(a, dtype=F32)
    if not self.offset:
      return _dev(torch, a)
    raw = torch.empty((a.size + 1,), device="cuda")
    self._keep.append(raw)
    v = raw[1:]
    v.copy_(torch.as_tensor(a))
    return v

  def struct(self, _lib):
    c = lambda a: ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))
    return _lib.OptOp(self.kind, len(self.shapes), c(self.arrays[0]), c(self.arrays[1]),
                      c(self.arrays[2]) if N_SLOTS[self.kind] >= 1 else None,
                      c(self.arrays[3]) if N_SLOTS[self.kind] >= 2 else None,
                      self.sizes, self.hyper_h, _ptr(self.step), c(self.arrays[4]), self.cols_h)

  def state(self):
    return ([_np(t).astype(np.float64) for t in self.p], [None if t is None else _np(t).astype(np.float64) for t in self.s0],
            [None if t is None else _np(t).astype(np.float64) for t in self.s1],
            None if self.step is None else int(self.step.item()))


def _check_opt(o, before, after, grads):
  """p, s0, s1 after one step against float64 TF1 rules evaluated on the state before it (and, for p, on the kernel's
  updated slots)"""
  (p0, a0, b0, st), (p1, a1, b1, _) = before, after
  h = o.hyper
  lr = h[0]
  for t in range(len(o.shapes)):
    g, p, pn = grads[t], p0[t], p1[t]
    tag = ["SGD", "Momentum", "RMSProp", "Adam", "cosine Momentum"][o.kind]
    if o.kind == SGD:
      _check(tag + " p", pn, p - lr * g, _gamma(2) * (np.abs(p) + np.abs(lr * g)))
    elif o.kind in (MOM, COS):
      m = h[1]
      _check(tag + " s0", a1[t], m * a0[t] + g, _gamma(2) * (np.abs(m * a0[t]) + np.abs(g)))
      dlr = 0.0
      if o.kind == COS:
        # fminf(step, decay_steps); 0.5 (1 + cosf(pi * st / ds)): the argument carries 3 roundings of pi (< 10 u),
        # cosf 2 ulp, 1 + cos; then ((1 - alpha) c + alpha) * lr: < 12 u lr in all
        ds, alpha = h[2], h[3]
        cs = 0.5 * (1 + np.cos(np.pi * min(st, ds) / ds))
        lr = h[0] * ((1 - alpha) * cs + alpha)
        dlr = 12 * U * h[0]
      upd = lr * a1[t]
      _check(tag + " p", pn, p - upd, _gamma(2) * (np.abs(p) + np.abs(upd)) + dlr * np.abs(a1[t]))
    elif o.kind == RMS:
      rho, mu, eps = h[1], h[2], h[3]
      # rho ms + ((1 - rho) g) g: (1 - rho) exact, three roundings
      _check(tag + " s0", a1[t], rho * a0[t] + (1 - rho) * g * g, _gamma(3) * (rho * a0[t] + (1 - rho) * g * g))
      q = lr * g / np.sqrt(a1[t] + eps)
      # lr g, ms + eps, sqrt, division, fused update: six roundings
      _check(tag + " s1", b1[t], mu * b0[t] + q, _gamma(6) * (np.abs(mu * b0[t]) + np.abs(q)))
      _check(tag + " p", pn, p - b1[t], _gamma(1) * (np.abs(p) + np.abs(b1[t])))
    else:
      b1_, b2_, eps = h[1], h[2], h[3]
      tt = st + 1
      P1, P2 = b1_ ** tt, b2_ ** tt
      lr_t = lr * np.sqrt(1 - P2) / (1 - P1)
      # powf <= 4 ulp relative to b^t, amplified by 1 / (1 - b^t) in the subtraction; sqrt halves it; sqrtf,
      # the product and the division: rel(lr_t) <= (4 P2/(1-P2) + 8 P1/(1-P1) + 6) u
      rel_lr = U * (4 * P2 / (1 - P2) + 8 * P1 / (1 - P1) + 6)
      _check(tag + " s0", a1[t], a0[t] + (1 - b1_) * (g - a0[t]),
             _gamma(3) * (np.abs(a0[t]) + (1 - b1_) * (np.abs(g) + np.abs(a0[t]))))
      _check(tag + " s1", b1[t], b0[t] + (1 - b2_) * (g * g - b0[t]),
             _gamma(4) * (np.abs(b0[t]) + (1 - b2_) * (g * g + np.abs(b0[t]))))
      upd = lr_t * a1[t] / (np.sqrt(b1[t]) + eps)
      # lr_t m, sqrtf(v), + eps, division: 4 u on top of rel(lr_t); then the subtraction
      _check(tag + " p", pn, p - upd, U * (np.abs(p) + np.abs(upd)) + 1.0001 * (rel_lr + 4 * U) * np.abs(upd))


def _opt_case(torch, _lib, lib, name, rng):
  """(optimizers of one adn_opt_step_group call, number of steps)"""
  if name in ("mixed", "offset"):
    starts = {SGD: None, MOM: 7, RMS: 0, ADAM: 0, COS: 1}     # the cosine decay passes decay_steps = 2.5 at step 3
    return [_Opt(torch, _lib, lib, rng, k, SHAPES, starts[k], name == "offset") for k in (SGD, MOM, RMS, ADAM, COS)], 4
  if name == "33_optimizers":
    ops = []
    for i in range(33):
      k = i % 5
      shapes = [SHAPES[(i + j) % len(SHAPES)] for j in range(1 + i % 3)]
      ops.append(_Opt(torch, _lib, lib, rng, k, shapes, (i if k in (ADAM, COS) or i % 2 else None), False))
    return ops, 3
  # 97 tensors: flushes after 96
  ops = []
  for i, nt in enumerate([32, 32, 32, 1]):
    k = (ADAM, MOM, COS, SGD)[i]
    ops.append(_Opt(torch, _lib, lib, rng, k, [SHAPES[(i + j) % len(SHAPES)] for j in range(nt)], 0, False))
  return ops, 3


@pytest.mark.parametrize("name", ["mixed", "offset", "33_optimizers", "97_tensors"])
def test_opt_step_group(env, name):
  """adn_opt_step_group over several steps: p, s0 and s1 within a few ulps of the float64 TF1 rules, each step counter
  +1 per call, and the hi / lo weight planes byte-identical to adn_planes_split of the updated parameters.  The
  optimizer does not refresh the sign bits: the GEMMs never read a weight's sign bits, so they are not compared."""
  torch, _lib, lib = env
  f16 = _lib.plane_format() == _lib.PLANES_F16
  rng = np.random.default_rng(len(name))
  opts, steps = _opt_case(torch, _lib, lib, name, rng)
  arr = (_lib.OptOp * len(opts))(*[o.struct(_lib) for o in opts])
  for _ in range(steps):
    grads = []
    for o in opts:
      gs = []
      for t, sh in enumerate(o.shapes):
        g = rng.standard_normal(int(np.prod(sh))).astype(F32)
        o.g[t].copy_(torch.as_tensor(g))
        gs.append(g.astype(np.float64))
      grads.append(gs)
    before = [o.state() for o in opts]
    _lib.check(lib.adn_opt_step_group(arr, len(opts), _sp(torch)), "adn_opt_step_group")
    for o, b, gs in zip(opts, before, grads):
      after = o.state()
      if o.step is not None:
        assert after[3] == b[3] + 1
      _check_opt(o, b, after, gs)
      for t, sh in enumerate(o.shapes):
        if o.planes[t] is None:
          continue
        hi_r, lo_r = _plane_regions(f16, sh[0], sh[1])
        got, ref = _bytes(o.planes[t]), _bytes(_split(torch, _lib, lib, o.p[t], sh[0], sh[1]))
        assert (got[hi_r] == ref[hi_r]).all() and (got[lo_r] == ref[lo_r]).all(), (o.kind, sh)
  assert not _lib.plane_overflow()


# ------------------------------------------------------------------------------------------------------------------
# a rejected call changes nothing
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("B", [300, 65537])
def test_head_group_failure_writes_nothing(env, B):
  """26 ops (two launches, or op by op above 512 CTAs); the last one's workspace is one byte short."""
  torch, _lib, lib = env
  C = 3
  inp, rng = _head_inputs(torch, B, C, 5)
  ops = _make_head_ops(torch, _lib, inp, rng, B, C, 26)
  ops[-1].ws_bytes = _lib.query(_lib.Q_HEAD_WS, B, C, ops[-1].N) - 257     # the query adds 256 B of slack
  outs = [t for o in ops for t in (o.out3, o.dw, o.dbias, o.dens, o.ens, o.planes) if t is not None]
  before = [_bytes(t) for t in outs]
  arr = (_lib.HeadOp * 26)(*[_head_struct(_lib, o) for o in ops])
  _lib.plane_overflow()
  rc = lib.adn_head_group(arr, 26, B, C, _sp(torch))
  msg = lib.adn_last_error().decode()
  torch.cuda.synchronize()
  assert all(np.array_equal(_bytes(t), b) for t, b in zip(outs, before))
  assert not _lib.plane_overflow()
  assert rc == ERR_WORKSPACE and "op 25:" in msg, msg


def test_bookkeeping_failure_writes_nothing(env):
  """130 entries (three launches); the last one has capacity 0."""
  torch, _lib, lib = env
  n = 130
  rng, caps, decays, ema, out3, sub, trace, books = _book_setup(torch, _lib, n, 3)
  for e in ema:
    e.copy_(torch.as_tensor(np.array([0.5, 2.0, 0.7], F32)))
  books[n - 1].capacity = 0
  step_d = torch.zeros((), dtype=torch.int64, device="cuda")
  outs = ema + trace
  before = [_bytes(t) for t in outs]
  rc = lib.adn_head_bookkeeping(books, n, step_d.data_ptr(), _sp(torch))
  msg = lib.adn_last_error().decode()
  torch.cuda.synchronize()
  assert all(np.array_equal(_bytes(t), b) for t, b in zip(outs, before))
  assert rc == ERR_INVALID and "entry 129:" in msg, msg


@pytest.mark.parametrize("name", ["33_optimizers", "97_tensors"])
def test_opt_group_failure_writes_nothing(env, name):
  """A call that flushes once; the last op has a null gradient pointer."""
  torch, _lib, lib = env
  rng = np.random.default_rng(9)
  opts, _ = _opt_case(torch, _lib, lib, name, rng)
  last = opts[-1]
  last.arrays[1][len(last.shapes) - 1] = None
  arr = (_lib.OptOp * len(opts))(*[o.struct(_lib) for o in opts])
  outs = [t for o in opts for ts in (o.p, o.s0, o.s1, o.planes) for t in ts if t is not None]
  outs += [o.step for o in opts if o.step is not None]
  before = [_bytes(t) for t in outs]
  rc = lib.adn_opt_step_group(arr, len(opts), _sp(torch))
  msg = lib.adn_last_error().decode()
  torch.cuda.synchronize()
  assert all(np.array_equal(_bytes(t), b) for t, b in zip(outs, before))
  assert rc == ERR_INVALID and ("op %d:" % (len(opts) - 1)) in msg, msg
