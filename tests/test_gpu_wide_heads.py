"""The wide head kernel (adn_head_group_wide) element-wise against a float64 restatement, in both plane formats, and
heads of more than 64 logits through the engine and the public API against the float64 oracle.

Error bounds follow the kernel's own summation order (csrc/heads.cu, ensemble_head_wide_kernel), with u = 2^-24 and
g(n) = n u / (1 - n u) the bound of a sequential fp32 sum of n terms:
  ens     bias + sum_k w_k m_k, one rounding per member:                 g(N + 1) * (|bias| + sum_k |w_k m_k|)
  row sums  a lane's 4-column chunks in sequence, then a 5-level xor tree: depth dr = 4 ceil(ceil(C/4) / 32) + 5
  softmax   a perturbation d of the logits moves p by <= 2 p max|d|; exp, the row sum and log add g(dr + 4)
  columns   rows of a row block in sequence, the blocks of a CTA in sequence, the finalize's lane-strided sum and
            5-level tree over the CTAs:                                   depth dcol = rb + bpc + ceil(n_cta/32) + 5
  loss      a warp's rows in sequence, the 8 warps, then the finalize:    depth rpw + 8 + ceil(n_cta/32) + 5
and the gradient errors of every summed term are added to the summation error."""

import ctypes
import math

import numpy as np
import pytest

from tests import parity_util as pu
from tests import wide_configs as wc
from tests.parity_util import orc

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 4 * 2.0 ** -149    # exp, x inv and x 1/B each round a subnormal result by up to 2^-150 absolute
SOFTMAX, MSE, SIGMOID = 0, 1, 2
SCALAR, VECTOR, MATRIX = 0, 1, 2


def gam(n):
  return n * U / (1 - n * U)


def wide_geom(batch, dim, members):
  """csrc/heads.cu wide_geom: rows per row block, row blocks per CTA, CTAs."""
  ld = (dim + 3) // 4 * 4
  rb = max(1, min(32, (96 * 1024) // (ld * 4)))
  nb = -(-batch // rb)
  cap = min(nb, max(64, min(512, (1 << 22) // (1 + dim + members * dim))))
  bpc = -(-nb // cap)
  return rb, bpc, -(-nb // bpc)


def wide_depths(batch, dim, members):
  rb, bpc, n_cta = wide_geom(batch, dim, members)
  dr = 4 * math.ceil(math.ceil(dim / 4) / 32) + 5
  fin = math.ceil(n_cta / 32) + 5
  return dict(dr=dr, dcol=rb + bpc + fin, dloss=bpc * math.ceil(rb / 8) + 8 + fin)


def narrow_depths(batch, dim, members):
  n_cta = math.ceil(batch / 128)
  fin = math.ceil(n_cta / 32) + 5
  return dict(dr=dim + 1, dcol=32 + 4 + fin, dloss=5 + 4 + fin)


@pytest.fixture(scope="module")
def lib():
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  eng._require_cuda()
  torch.manual_seed(0)
  return _lib.load()


class Op:
  """One adn_head_op with its device inputs and outputs (torch tensors) and its float64 restatement."""

  def __init__(self, torch, members, head, mix, w, bias, gammas, labels, labels_f, grads=True, dens=True, ens_out=False,
               planes=False, colsum_only=False, dz=0, reg_is_zero=False, narrow=False):
    from adanet_b200 import _lib
    self.torch, self.members, self.head, self.mix, self.w, self.bias = torch, members, head, mix, w, bias
    self.gammas, self.labels, self.labels_f, self.colsum_only, self.dz = gammas, labels, labels_f, colsum_only, dz
    self.reg_is_zero = reg_is_zero or colsum_only
    B, C = members[0].shape
    N = len(members)
    self.B, self.C, self.N = B, C, N
    dev = members[0].device
    f32 = dict(dtype=torch.float32, device=dev)
    self.out3 = torch.empty(3, **f32)
    self.dw = torch.empty(w.shape, **f32) if (grads and not colsum_only and mix != MATRIX and w is not None) else None
    if grads and not colsum_only and mix != MATRIX and w is None:
      self.dw = torch.empty((N,) if mix == SCALAR else (N, C), **f32)
    self.dbias = torch.empty(C, **f32) if grads else None
    self.dens = torch.empty((B, C), **f32) if dens else None
    self.ens_out = torch.empty((B, C), **f32) if ens_out else None
    self.planes = torch.empty(_lib.query(_lib.Q_PLANES_BYTES, B, C), dtype=torch.uint8, device=dev) if planes else None
    q = _lib.Q_HEAD_WS if narrow else _lib.Q_HEAD_WIDE_WS
    self.ws = torch.empty(_lib.query(q, B, C, N), dtype=torch.uint8, device=dev)
    self.plane_region = _plane_region(_lib.plane_format(), B, C)
    self._m = _lib.ptr_array([m.data_ptr() for m in members])
    self._g = _lib.f32_array(gammas)
    ptr = lambda t: t.data_ptr() if t is not None else None
    self.op = _lib.HeadOp(head, mix, ctypes.cast(self._m, ctypes.POINTER(ctypes.c_void_p)), N, int(self.reg_is_zero),
                          ptr(w), ptr(bias), ctypes.cast(self._g, ctypes.POINTER(ctypes.c_float)), 2.0, dz, ptr(labels),
                          ptr(labels_f), ptr(self.out3), ptr(self.dw), ptr(self.dbias), ptr(self.dens), ptr(self.ens_out),
                          ptr(self.planes), int(colsum_only), 0, ptr(self.ws), self.ws.numel())

  def outputs(self):
    return [t for t in (self.out3, self.dw, self.dbias, self.dens, self.ens_out, self.planes) if t is not None]

  def fill(self, byte=0xFF):
    for t in self.outputs():
      t.view(self.torch.uint8).fill_(byte)

  def snapshot(self):
    """Every output byte the kernel writes (of the planes: both planes' rows, not the sign bits or the tail)."""
    out = [t.clone() for t in self.outputs() if t is not self.planes]
    if self.planes is not None:
      written, one = self.plane_region
      out += [self.planes[:written].clone(), self.planes[one:one + written].clone()]
    return out

  def check(self, depths):
    """Every output against the float64 restatement within the bounds of the module docstring."""
    torch = self.torch
    B, C, N = self.B, self.C, self.N
    d64 = lambda t: t.double()
    unit = self.mix == MATRIX or self.w is None
    e = d64(self.bias).expand(B, C).clone() if self.bias is not None else torch.zeros((B, C), dtype=torch.float64,
                                                                                          device=self.out3.device)
    S = e.abs()
    for k, m in enumerate(self.members):
      wk = 1.0 if unit else (d64(self.w[k]) if self.mix == SCALAR else d64(self.w[k])[None, :])
      t = wk * d64(m)
      e += t
      S += t.abs()
    E = gam(N + 1) * S
    dr, dcol, dloss = depths["dr"], depths["dcol"], depths["dloss"]
    if self.head == SOFTMAX:
      y = self.labels.long()
      lse = torch.logsumexp(e, 1)
      p = torch.exp(e - lse[:, None])
      loss_r = lse - e.gather(1, y[:, None])[:, 0]
      onehot = torch.zeros_like(e).scatter_(1, y[:, None], 1.0)
      g = (p - onehot) / B
      er = E.max(1).values[:, None]
      dG = p * (2 * er + gam(dr + 4)) / B + 3 * U * g.abs() + TINY
      dL = 3 * er[:, 0] + gam(dr + 6) * (1 + loss_r.abs() + math.log(C))
      denom = B
    else:
      z = d64(self.labels_f)
      if self.head == MSE:
        d = e - z
        el = d * d
        g = 2 * d / (B * C)
        dd = E + U * d.abs()
        dL = (2 * d.abs() * dd + dd * dd + 2 * U * el).sum(1) + gam(dr) * el.sum(1)
        dG = 2 * dd / (B * C) + 4 * U * g.abs() + TINY
      else:
        el = torch.clamp(e, min=0) - e * z + torch.log1p(torch.exp(-e.abs()))
        g = (torch.sigmoid(e) - z) / (B * C)
        dL = (E * (1 + z.abs()) + gam(4) * (torch.clamp(e, min=0) + (e * z).abs() + el.abs()) + 4 * U).sum(1) + \
            gam(dr) * el.abs().sum(1)
        dG = (E / 4 + 4 * U) / (B * C) + 4 * U * g.abs() + TINY
      loss_r = el.sum(1)
      denom = B * C
    loss = loss_r.sum() / denom
    dloss_b = float((dL.sum() + gam(dloss) * loss_r.abs().sum()) / denom + 3 * U * abs(float(loss)))
    # regulariser
    if self.reg_is_zero:
      reg, dreg = 0.0, 0.0
    else:
      wdim = 1 if self.mix == SCALAR else C
      terms = []
      for k in range(N):
        if self.mix == MATRIX:
          l1 = float(self.w[k])
        elif self.w is None:
          l1 = float(wdim)
        else:
          l1 = float(d64(self.w[k]).abs().sum())
        terms.append(self.gammas[k] * l1)
      reg = float(np.sum(terms))
      dreg = gam(N + wdim + 2) * float(np.sum(np.abs(terms)))
    self._close("loss", self.out3[0], loss, dloss_b)
    if not self.colsum_only:
      self._close("reg", self.out3[1], reg, dreg)
      self._close("adanet_loss", self.out3[2], float(loss) + reg, dloss_b + dreg + U * abs(float(loss) + reg))
    if self.ens_out is not None:
      self._close("ens_out", self.ens_out, e, E)
    if self.dens is not None:
      self._close("dens", self.dens, g, dG)
    if self.dbias is not None:
      self._close("dbias", self.dbias, g.sum(0), dG.sum(0) + gam(dcol) * g.abs().sum(0))
    if self.dw is not None:
      want, bound = [], []
      for k, m in enumerate(self.members):
        gm = g * d64(m)
        err = dG * d64(m).abs()
        if self.mix == SCALAR:
          want.append(gm.sum())
          bound.append(err.sum() + gam(dr + dcol + 1) * gm.abs().sum())
        else:
          want.append(gm.sum(0))
          bound.append(err.sum(0) + gam(dcol + 1) * gm.abs().sum(0))
      want, bound = torch.stack(want), torch.stack(bound)
      if not self.reg_is_zero:
        wv = d64(self.w) if self.w is not None else torch.ones_like(want)
        gk = torch.tensor(self.gammas, dtype=torch.float64, device=want.device)
        r = 2.0 * (gk if self.mix == SCALAR else gk[:, None]) * torch.sign(wv)
        want, bound = want + r, bound + 3 * U * r.abs()
      self._close("dw", self.dw, want, bound + U * want.abs())
    return g

  @staticmethod
  def _close(name, got, want, bound):
    import torch
    got = got.double()
    want = torch.as_tensor(want, dtype=torch.float64, device=got.device)
    bound = torch.as_tensor(bound, dtype=torch.float64, device=got.device)
    err = (got - want).abs()
    bad = ~(err <= bound + 1e-300)
    if bool(bad.any()):
      i = int(bad.flatten().nonzero()[0])
      raise AssertionError("%s: %d elements off; first at %d: got %r want %r bound %r" % (
          name, int(bad.sum()), i, float(got.flatten()[i]), float(want.flatten()[i]),
          float(bound.expand_as(err).flatten()[i])))


def _inputs(torch, B, C, N, misalign=False, seed=0):
  gen = torch.Generator(device="cuda").manual_seed(seed)
  dev = torch.device("cuda")
  if misalign:
    # every member row starts 4 bytes past a 16 B boundary: the scalar-load path at a dim that allows 16 B loads
    buf = torch.randn((N, B * C + 1), generator=gen, device=dev) * 2
    members = [buf[k, 1:].view(B, C) for k in range(N)]
  else:
    members = [torch.randn((B, C), generator=gen, device=dev) * 2 for _ in range(N)]
  labels = torch.randint(0, C, (B,), generator=gen, device=dev)
  labels_f = torch.rand((B, C), generator=gen, device=dev)
  w_s = torch.rand((N,), generator=gen, device=dev) * 2 - 1
  w_v = torch.rand((N, C), generator=gen, device=dev) * 2 - 1
  l1 = torch.rand((N,), generator=gen, device=dev) * 3
  bias = torch.randn((C,), generator=gen, device=dev) * 0.5
  gammas = [0.01 * (k + 1) for k in range(N)]
  return members, labels, labels_f, w_s, w_v, l1, bias, gammas


def _ops(torch, B, C, N, misalign=False, overflow=False):
  members, labels, labels_f, w_s, w_v, l1, bias, gammas = _inputs(torch, B, C, N, misalign)
  dz_big = 30 if overflow else 0
  return [
      Op(torch, members, SOFTMAX, SCALAR, w_s, None, gammas, labels, None, ens_out=True, planes=True),
      Op(torch, members, SOFTMAX, VECTOR, None, bias, gammas, labels, None, reg_is_zero=True),
      Op(torch, members, MSE, MATRIX, l1, bias, gammas, None, labels_f, planes=True, dz=dz_big),
      Op(torch, members, SIGMOID, VECTOR, w_v, None, gammas, None, labels_f, dens=False, ens_out=True),
      Op(torch, members[:1], SOFTMAX, SCALAR, None, None, [0.0], labels, None, colsum_only=True, planes=True, dz=-3),
      Op(torch, members, MSE, SCALAR, w_s, bias, gammas, None, labels_f, grads=False, dens=False, ens_out=True),
      Op(torch, members, SIGMOID, SCALAR, None, bias, gammas, None, labels_f),
      Op(torch, members[:1], SIGMOID, SCALAR, None, None, [0.0], None, labels_f, colsum_only=True, planes=True),
      Op(torch, members[:1], MSE, SCALAR, None, None, [0.0], None, labels_f, colsum_only=True, dens=True),
  ]


def _call(lib, ops, B, C, wide=True):
  from adanet_b200 import _lib
  arr = (_lib.HeadOp * len(ops))(*[o.op for o in ops])
  f = lib.adn_head_group_wide if wide else lib.adn_head_group
  return f(arr, len(ops), B, C, None)


def _plane_region(fmt, B, C):
  bk, es = (64, 2) if fmt == 1 else (32, 4)
  written = B * math.ceil(C / bk) * bk * es
  one = (B * math.ceil(C / bk) * bk + 127) // 128 * 128 * es
  return written, one


@pytest.fixture(params=["f16", "tf32"])
def fmt(request, lib):
  from adanet_b200 import _lib
  f = _lib.PLANES_F16 if request.param == "f16" else _lib.PLANES_TF32
  old = _lib.plane_format()
  _lib.set_plane_format(f)
  yield f
  _lib.set_plane_format(old)


# (C, N, batch, misaligned members, full checks: many-op vs alone, rerun, rejected call, graph replay)
SHAPES = [
    (65, 1, 1, False, True), (65, 64, 129, False, False), (100, 2, 1000, True, True), (100, 8, 32768, False, False),
    (127, 8, 65537, False, False), (1000, 64, 129, False, False), (1000, 1, 65537, False, False),
    (1000, 8, 1000, False, True), (4096, 2, 1000, False, False), (4096, 1, 32768, False, False),
]


@pytest.mark.parametrize("C,N,B,misalign,full", SHAPES, ids=["C%d-N%d-B%d" % s[:3] for s in SHAPES])
def test_wide_head_kernel_matches_fp64(lib, fmt, C, N, B, misalign, full):
  import torch
  from adanet_b200 import _lib
  ops = _ops(torch, B, C, N, misalign, overflow=(B == 1000))
  for o in ops:
    o.fill()
  _lib.plane_overflow()                                         # clear the sticky flag
  _lib.check(_call(lib, ops, B, C), "adn_head_group_wide")
  flag = _lib.plane_overflow()
  torch.cuda.synchronize()
  for o in ops:
    o.check(wide_depths(B, C, o.N))
  # planes: byte-identical to adn_planes_split_scaled of the kernel's own dens, padding columns included; the flag
  # raised exactly when a scaled value does not fit fp16
  written, one = _plane_region(fmt, B, C)
  want_flag = False
  for o in ops:
    if o.planes is None:
      continue
    ref = torch.zeros_like(o.planes)
    _lib.check(lib.adn_planes_split_scaled(o.dens.data_ptr(), B, C, ref.data_ptr(), o.dz, None), "split")
    torch.cuda.synchronize()
    for off in (0, one):
      assert torch.equal(o.planes[off:off + written], ref[off:off + written])
    m = (o.dens.double() * 2.0 ** o.dz).abs()
    want_flag |= bool(((m >= 65520) & torch.isfinite(m)).any()) and fmt == _lib.PLANES_F16
  assert flag == want_flag
  if not full:
    return
  first = [o.snapshot() for o in ops]
  # a second run of the same call: byte-identical
  for o in ops:
    o.fill(0x7F)
  _lib.check(_call(lib, ops, B, C), "adn_head_group_wide")
  for o, s in zip(ops, first):
    assert all(torch.equal(a, b) for a, b in zip(o.snapshot(), s))
  # each op alone: byte-identical to the many-op call
  for o, s in zip(ops, first):
    o.fill(0x3F)
    _lib.check(_call(lib, [o], B, C), "adn_head_group_wide")
    assert all(torch.equal(a, b) for a, b in zip(o.snapshot(), s))
  # a rejected call (its last op has 65 members) writes nothing
  bad = Op(torch, ops[0].members, SOFTMAX, SCALAR, None, None, [0.0] * N, ops[0].labels, None)
  bad.op.n_members = 65
  for o in ops:
    o.fill(0x11)
  sentinel = [o.snapshot() for o in ops]
  assert _call(lib, ops + [bad], B, C) == -95
  torch.cuda.synchronize()
  for o, s in zip(ops, sentinel):
    assert all(torch.equal(a, b) for a, b in zip(o.snapshot(), s))
  # CUDA-graph replay: the same bytes as the eager launches
  stream = torch.cuda.Stream()
  g = torch.cuda.CUDAGraph()
  from adanet_b200 import _lib as L
  with torch.cuda.graph(g, stream=stream):
    arr = (L.HeadOp * len(ops))(*[o.op for o in ops])
    L.check(lib.adn_head_group_wide(arr, len(ops), B, C, torch.cuda.current_stream().cuda_stream), "capture")
  for o in ops:
    o.fill(0x22)
  g.replay()
  torch.cuda.synchronize()
  for o, s in zip(ops, first):
    assert all(torch.equal(a, b) for a, b in zip(o.snapshot(), s))


@pytest.mark.parametrize("C,N", [(10, 2), (33, 4)])
def test_wide_agrees_with_narrow_kernel(lib, fmt, C, N):
  """Where both kernels run, each meets its own bounds against fp64 and the two agree within the sum of them."""
  import torch
  from adanet_b200 import _lib
  B = 1000
  members, labels, labels_f, w_s, w_v, l1, bias, gammas = _inputs(torch, B, C, N, seed=5)
  mk = lambda narrow: [Op(torch, members, SOFTMAX, VECTOR, w_v, bias, gammas, labels, None, ens_out=True, narrow=narrow),
                       Op(torch, members, MSE, SCALAR, w_s, None, gammas, None, labels_f, narrow=narrow),
                       Op(torch, members, SIGMOID, MATRIX, l1, bias, gammas, None, labels_f, narrow=narrow)]
  nar, wid = mk(True), mk(False)
  _lib.check(_call(lib, nar, B, C, wide=False), "adn_head_group")
  _lib.check(_call(lib, wid, B, C), "adn_head_group_wide")
  torch.cuda.synchronize()
  for a, b in zip(nar, wid):
    a.check(narrow_depths(B, C, N))
    b.check(wide_depths(B, C, N))
    for x, y in zip(a.outputs(), b.outputs()):
      d = (x.double() - y.double()).abs().max()
      assert float(d) < 1e-4 * max(1.0, float(x.double().abs().max())), float(d)


# ---- engine and public API ----

def _check_runs(o_res, reps, tol=1e-5):
  worst = 0.0
  for o, r in zip(o_res, reps):
    assert r.candidate_names == o.candidate_names
    for name, tr in o.traces.items():
      for f in ("sub_loss", "ens_loss", "adanet_loss", "ema"):
        err = np.abs(r.traces[name][f].astype(np.float64) - np.asarray(tr[f], dtype=np.float64)).max()
        worst = max(worst, err)
        assert err < tol, "iteration %d %s/%s: max abs err %.3g" % (o.iteration, name, f, err)
    assert r.best_index == o.best_index, (r.ema_losses, o.ema_losses)
    assert r.architecture == o.architecture
    np.testing.assert_allclose(r.ema_losses, o.ema_losses, atol=tol)
  return worst


@pytest.mark.parametrize("name", sorted(wc.CONFIGS))
def test_wide_head_search_parity(lib, name):
  from adanet_b200 import _lib
  cfg = wc.CONFIGS[name]
  o = wc.oracle_run(cfg)
  r, s = wc.engine_run(cfg)
  worst = _check_runs(o, r)
  print("%s worst per-step abs err %.3g" % (name, worst))
  if name == "c48_force_grow":
    n = [len(rep.architecture) for rep in r]
    assert n[-1] == cfg["iters"]
    # the grown ensemble head left the narrow kernel partway through; the subnetwork losses never did
    assert _lib.query(_lib.Q_HEAD_PATH, 48, 2) == 0 and _lib.query(_lib.Q_HEAD_PATH, 48, cfg["iters"]) == 1
    assert _lib.query(_lib.Q_HEAD_PATH, 48, 1) == 0


def test_head_wider_than_any_kernel_refused_at_plan_build(lib):
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  specs = pu.make_specs([(1, 8)], 8, 16385, 0, ("sgd", 0.01))[1]
  before = _lib.launch_count()
  with pytest.raises(NotImplementedError, match="16385 logits"):
    eng.IterationPlan(0, specs, [], eng.EnsemblerPlanSpec(**wc.ENS), 32, 8, 16385)
  assert _lib.launch_count() == before


def test_simple_cnn_100_classes_parity(lib):
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  from tests.test_gpu_iteration import CNN_CASES, _cnn_data
  case = dict(CNN_CASES["cifar_shaped"], steps=8)
  C = 100
  x, y = _cnn_data(case, classes=C)
  opt = case["opt"](case["steps"])
  mk = lambda t, which: pu.make_cnn_specs(case["seeds"], case["image"], case["filters"], case["hidden"], C, t, opt)[which]
  o, _ = orc.run_adanet(lambda t, frozen: mk(t, 0), x, y, case["B"], case["steps"], case["iters"], orc.EnsemblerSpec(),
                        C, adanet_loss_decay=0.99)
  s = srch.AdaNetSearch(lambda t, frozen: mk(t, 1), eng.EnsemblerPlanSpec(), int(np.prod(case["image"])), C, case["B"],
                        adanet_loss_decay=0.99)
  reps = s.run(srch.consecutive_batches(x, y, case["B"]), case["steps"], case["iters"])
  print("cnn 100 classes worst per-step abs err %.3g" % _check_runs(o, reps))


def test_estimator_100_classes_lifecycle(lib, tmp_path):
  """MultiClassHead(100) through Estimator: two iterations matching the oracle's selection and per-step losses,
  evaluate on a ragged hold-out, predict [n, 100] probabilities, and a resume from a mid-iteration checkpoint that
  ends bit-identical to the uninterrupted run."""
  import adanet_b200 as adanet
  from adanet_b200 import graph, train
  from adanet_b200.examples import simple_dnn
  from tests import test_gpu_api as api
  B, D, C, SEED = 128, 20, 100, 7
  x, y = orc.make_tabular(B * 40, D, C, seed=4321)
  steps, iters, lr = 10, 2, 0.05

  def space(t, frozen):
    depth = 0 if not frozen else len(frozen[-1].ws) - 1
    specs = []
    for nl in (depth, depth + 1):
      dims = [D] + [16] * nl + [C]
      ws = [api._glorot((dims[i], dims[i + 1]), SEED) for i in range(len(dims) - 1)]
      bs = [np.zeros((d,), np.float32) for d in dims[1:]]
      specs.append(orc.SubnetworkSpec("linear" if nl == 0 else "{}_layer_dnn".format(nl), dims,
                                      float(np.sqrt(np.float32(nl))), ("sgd", lr), ws=ws, bs=bs))
    return specs

  def input_fn(xx, yy, start=0, tail=0):
    def fn():
      for i in range(start * B, xx.shape[0] - B + 1, B):
        yield {"x": xx[i:i + B]}, yy[i:i + B]
      if tail:
        yield {"x": xx[-tail:]}, yy[-tail:]
    return fn

  def make(model_dir, save=None):
    gen = api._modern(simple_dnn.Generator(feature_columns=[graph.numeric_column("x", D)],
                                           optimizer=train.GradientDescentOptimizer(lr), layer_size=16, seed=SEED))
    kw = dict(config=adanet.RunConfig(model_dir=model_dir, save_checkpoints_steps=save)) if save else {}
    return adanet.Estimator(
        head=adanet.heads.MultiClassHead(C), subnetwork_generator=gen, max_iteration_steps=steps,
        ensemblers=[adanet.ensemble.ComplexityRegularizedEnsembler(optimizer=train.GradientDescentOptimizer(0.01),
                                                                   adanet_lambda=0.01, adanet_beta=0.001)],
        max_iterations=iters, model_dir=model_dir, debug=True, **kw)

  est = make(str(tmp_path / "full"), save=3)
  est.train(input_fn(x, y), max_steps=steps * iters)
  ens = orc.EnsemblerSpec(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001)
  results, frozen = orc.run_adanet(space, x, y, B, steps, iters, ens, C)
  for rep, res in zip(est._search.reports, results):
    assert rep.best_index == res.best_index and rep.architecture == res.architecture
    np.testing.assert_allclose(rep.ema_losses, res.ema_losses, atol=1e-5, rtol=0)
    for name, tr in res.traces.items():
      np.testing.assert_allclose(rep.traces[name]["sub_loss"], tr["sub_loss"], atol=1e-5, rtol=0)
      np.testing.assert_allclose(rep.traces[name]["adanet_loss"], tr["adanet_loss"], atol=1e-5, rtol=0)
  # ragged hold-out: two full batches and a 37-example tail
  xe, ye = orc.make_tabular(B * 2 + 37, D, C, seed=99)
  ev = est.evaluate(input_fn(xe, ye, tail=37))
  mw, bias = results[-1].mixture_weights, results[-1].bias

  def oracle_eval(xb, yb):
    logits = [orc.mlp_forward(m.ws, m.bs, xb)[-1] for m in frozen]
    e = orc.ensemble_logits("scalar", list(mw), bias, logits, [None] * len(logits))
    return float(orc.softmax_xent_mean(e, yb)[0]), e

  parts = [(xe[i:i + B], ye[i:i + B]) for i in (0, B)] + [(xe[-37:], ye[-37:])]
  losses = [oracle_eval(a, b) for a, b in parts]
  assert abs(ev["loss"] - np.mean([l for l, _ in losses])) < 1e-5
  correct = sum(int((np.argmax(e, 1) == b).sum()) for (_, e), (_, b) in zip(losses, parts))
  assert abs(ev["accuracy"] - correct / (2 * B + 37)) < 1e-9
  preds = list(est.predict(input_fn(xe[:B], ye[:B])))
  probs = np.stack([p["probabilities"] for p in preds])
  assert probs.shape == (B, C)
  e0 = losses[0][1]
  want = np.exp(e0 - e0.max(1, keepdims=True))
  np.testing.assert_allclose(probs, want / want.sum(1, keepdims=True), atol=2e-6)
  # killed inside iteration 1, resumed from the last in-flight checkpoint (global step 12)
  a = make(str(tmp_path / "killed"), save=3)
  a.train(input_fn(x, y), max_steps=14)
  b = make(str(tmp_path / "killed"), save=3)
  b.train(input_fn(x, y, start=12), max_steps=steps * iters)
  ra, rb = est._search.reports[-1], b._search.reports[-1]
  assert rb.best_index == ra.best_index and rb.architecture == ra.architecture
  np.testing.assert_array_equal(rb.ema_losses, ra.ema_losses)
  np.testing.assert_array_equal(rb.mixture_weights, ra.mixture_weights)
