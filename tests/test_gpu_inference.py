"""The inference path element by element against float64: EnsembleEvalPlan (Estimator.evaluate / predict and the
Evaluator's `previous_ensemble`), IterationPlan.eval_step (the Evaluator's candidate ranking) and what evaluate /
predict make of them on the host.

The float64 reference restates every member's forward (conv stem included) and carries a componentwise error bound
through it: each layer adds TOL (|h| + E) |W| + TOL |b| for its own rounding (the fp32 dot-product bound (K + 2) U on
the SIMT path), plus the fp16 planes' 2^-36 floor, and passes E |W| on (ReLU is 1-Lipschitz).  The ensemble logits
add 2 (N + 1) U of rounding to sum_k |w_k| E_k, and the head's loss bound follows from that (test_gpu_step_state).

  EnsembleEvalPlan  injected weights; SCALAR / VECTOR / MATRIX mixture weights with and without bias, lambda = beta = 0
                    or not, MATRIX over a linear member (its last layer is the input planes), a MeanEnsemble winner
                    (previous members weigh 0), 1 / 3 / 8 members of depth 0..8 and widths around 64 and 128, a
                    SimpleCNN member beside dense ones, the three heads, B in {1, 37, 128, 129, 4097}; ens_logits and
                    out3 within their bounds, `y=None` gives the same logits, a second run the same bytes, the members
                    are left byte-identical, and a partial batch evaluates its own rows
  eval_step         all four metrics of every candidate ensemble after two training steps, on a full and a partial
                    batch; a dropout candidate evaluates without its mask; the training state is left byte-identical
  Estimator         evaluate / predict over an input with a ragged tail, against float64 of ensemble-latest.npz; a
                    fresh Estimator predicts the same bytes; an Evaluator with a ragged hold-out set ranks every
                    candidate and the previous ensemble by their float64 values
  format switch     the eval plan the Estimator hands out after a switch to TF32 planes has buffers of that format

The worst err/bound of every check is printed at the end of the module (pytest -s).
"""

import json
import os

import numpy as np
import pytest

from tests.parity_util import orc
from tests.test_gpu_plane_groups import _cw, _open, _set_format
from tests.test_gpu_step_state import (CASES, F16_FLOOR, U, _build_plan, _case_data, _members, conv_stem64, f64,
                                       head_loss, layer_fwd)

D = 100
REPORT = {}
_PATH = ["f16"]             # the path of the test running: f16 / tf32 planes or the fp32 SIMT path


def _check(fails, check, got, exact, bound, what):
  got = np.asarray(got)
  exact, bound = np.broadcast_to(f64(exact), got.shape), np.broadcast_to(f64(bound), got.shape)
  err = np.abs(f64(got) - exact)
  if err.size:
    r = float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), np.where(err > 0, np.inf, 0.0))))
    REPORT[(_PATH[0], check)] = max(REPORT.get((_PATH[0], check), 0.0), r)
  fails += _cw(got, exact, bound, what)


@pytest.fixture(scope="module", autouse=True)
def _print_report():
  yield
  for p in sorted({p for p, _ in REPORT}):
    print("\n%s: " % p + ", ".join("%s %.3g" % (c, v) for (pp, c), v in sorted(REPORT.items()) if pp == p))


@pytest.fixture(params=["f16", "tf32"])
def fmt(request):
  """f16 or tf32 planes, for the tests that run the plane path only"""
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _set_format(_lib, request.param)
  _lib.plane_overflow()
  _PATH[0] = request.param
  try:
    yield request.param
  finally:
    _lib.set_plane_format(before)


# ------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------
def member64(ws, bs, x, image=None, floor=0.0, fp32_dot=False):
  """float64 (logits, their bound, last layer, its bound) of one member from its weights (a conv stem's HWIO kernel
  first when `image` = (H, W, Cin)), with the componentwise error bound carried layer by layer.  The last layer is the
  input to the logits layer: the last hidden activation, the pooled features, or x itself for a linear model."""
  h = f64(x)
  E = np.zeros_like(h)
  if image is not None:
    st = conv_stem64(h.reshape((-1,) + tuple(image)), ws[0], bs[0])
    h, E = st["pooled"], st["bound"] + floor
    ws, bs = ws[1:], bs[1:]
  for i, (w, b) in enumerate(zip(ws, bs)):
    last = i == len(ws) - 1
    if last:
      lh, lE = h, E
    z, _ = layer_fwd(h, w, b, not last)
    _, own = layer_fwd(np.abs(h) + E, np.abs(f64(w)), np.abs(f64(b)), False, floor=floor, fp32_dot=fp32_dot)
    E = own + E @ np.abs(f64(w))
    h = z
  return h, E, lh, lE


def ensemble64(head, mix, w, bias, logits, errs, y, gammas):
  """float64 ensemble logits, their bound, out3 = (loss, reg, adanet_loss) and its bound over the members' logits
  with their errors.  mix "scalar" w [N] / "vector" w [N, C]; "matrix": `logits` are the members' last layers times
  W_k and w is the list of the W_k.  y None: out3 is None."""
  N = len(logits)
  bias = f64(bias)
  if mix == "matrix":
    wk = [1.0] * N
    l1 = [np.abs(f64(W)).sum() for W in w]
    size = sum(np.size(W) for W in w)
  else:
    wk = [f64(w)[k] for k in range(N)]
    l1 = [np.abs(v).sum() for v in wk]
    size = np.size(w)
  e = bias + sum(a * m for a, m in zip(wk, logits))
  e_err = 2 * (N + 1) * U * (np.abs(bias) + sum(np.abs(a * m) for a, m in zip(wk, logits)))
  e_err = e_err + sum(np.abs(a) * E for a, E in zip(wk, errs))
  if y is None:
    return e, e_err, None, None
  loss, lb, _, _ = head_loss(head, e, y, e_err)
  reg = float(sum(g * v for g, v in zip(gammas, l1)))
  reg_b = 2 * (size + N) * U * reg
  out3 = np.array([loss, reg, loss + reg])
  return e, e_err, out3, np.array([lb, reg_b, lb + reg_b]) + 4 * U * np.abs(out3)


def gamma32(lam, beta, cx):
  """weighted.py:351-358 in fp32: lambda * r(h) + beta, or beta alone when lambda = 0"""
  lam, beta = np.float32(lam), np.float32(beta)
  return float(beta if lam == 0.0 else np.float32(lam * np.float32(cx) + beta))


def ambiguous(head, e, e_err):
  """rows whose predicted class the engine may legitimately flip: a softmax row whose top-2 margin is within twice
  the bound, a sigmoid logit within its bound of 0"""
  if head == "softmax_xent":
    top = np.sort(e, axis=1)
    return (top[:, -1] - top[:, -2]) <= 2 * e_err.max(axis=1)
  return (np.abs(e) <= e_err).reshape(-1)


def correct64(head, e, y):
  if head == "softmax_xent":
    return e.argmax(axis=1) == np.asarray(y).reshape(-1)
  return ((e > 0) == (f64(y) > 0.5)).reshape(-1)


def check_accuracy(fails, head, got, e, e_err, y, what):
  """got = the correct share of the examples (over several batches: of all their examples), against float64
  where the prediction is clear; an ambiguous example may count either way"""
  ok, amb = correct64(head, e, y), ambiguous(head, e, e_err)
  lo, hi = float((ok & ~amb).sum()) / ok.size, float((ok | amb).sum()) / ok.size
  REPORT[(_PATH[0], "accuracy: ambiguous share")] = max(REPORT.get((_PATH[0], "accuracy: ambiguous share"), 0.0),
                                                        float(amb.mean()))
  if not lo - 1e-12 <= got <= hi + 1e-12:
    fails.append("%s: accuracy %r outside [%r, %r] (%d ambiguous of %d)" % (what, got, lo, hi, int(amb.sum()), amb.size))


# ------------------------------------------------------------------------------------------------------------------
# EnsembleEvalPlan with injected weights
# ------------------------------------------------------------------------------------------------------------------
LAM = (0.02, 0.003)
WB_CASES = {
    "scalar_b1": dict(B=1, C=10, head="softmax_xent", mix="scalar", members=[[D, 10]]),
    "scalar_bias_reg_b37": dict(B=37, C=10, head="softmax_xent", mix="scalar", bias=True, reg=LAM,
                                members=[[D, 10], [D, 63, 10], [D, 129, 65, 10]]),
    "vector_b128_c33": dict(B=128, C=33, head="softmax_xent", mix="vector", members=[[D, 64, 33], [D, 33], [D, 128, 127, 33]]),
    "vector_bias_reg_8_b129_c2": dict(B=129, C=2, head="softmax_xent", mix="vector", bias=True, reg=LAM,
                                      members=[[D] + [65] * d + [2] for d in range(8)]),
    "deep8_b4097": dict(B=4097, C=10, head="softmax_xent", mix="scalar", bias=True, reg=LAM,
                        members=[[D] + [24] * 8 + [10], [D, 10], [D, 129, 64, 10]]),
    "matrix_b129": dict(B=129, C=10, head="softmax_xent", mix="matrix", members=[[D, 10], [D, 48, 10], [D, 40, 130, 72, 10]]),
    "matrix_bias_reg_b37": dict(B=37, C=10, head="softmax_xent", mix="matrix", bias=True, reg=LAM,
                                members=[[D, 10], [D, 65, 10], [D, 127, 129, 10]]),
    "matrix_mse_b128": dict(B=128, C=3, head="mse", mix="matrix", bias=True, reg=LAM, members=[[D, 3], [D, 64, 64, 3]]),
    "mean_b128": dict(B=128, C=10, head="softmax_xent", mix="scalar", mean=2, members=[[D, 10], [D, 32, 10], [D, 64, 10],
                                                                                      [D, 40, 24, 10]]),
    "mse_c1_b129": dict(B=129, C=1, head="mse", mix="scalar", members=[[D, 1], [D, 40, 1], [D, 65, 127, 1]]),
    "mse_vector_bias_reg_b37": dict(B=37, C=3, head="mse", mix="vector", bias=True, reg=LAM, members=[[D, 3], [D, 40, 72, 3]]),
    "sigmoid_c1_vector_bias_reg_b128": dict(B=128, C=1, head="sigmoid_xent", mix="vector", bias=True, reg=LAM,
                                            members=[[D, 20, 1], [D, 1], [D, 129, 1]]),
    "sigmoid_c2_b1": dict(B=1, C=2, head="sigmoid_xent", mix="scalar", reg=LAM, members=[[D, 40, 2], [D, 2]]),
    # a SimpleCNN member (8x8x3 images, 16 filters: 256 pooled features) beside dense members on the flattened images
    "cnn_scalar_bias_b128": dict(B=128, C=10, head="softmax_xent", mix="scalar", bias=True, reg=LAM, input=192,
                                 members=[dict(dims=[256, 32, 10], image=(8, 8, 3)), [192, 10], [192, 65, 10]]),
    # MATRIX over a linear SimpleCNN member: its last layer is the pooled features
    "cnn_matrix_b37": dict(B=37, C=10, head="softmax_xent", mix="matrix", bias=True, reg=LAM, input=192,
                           members=[dict(dims=[256, 10], image=(8, 8, 3)), [192, 10], [192, 40, 10]]),
}
SIMT_WB = sorted(k for k, c in WB_CASES.items() if c["mix"] != "matrix" and c.get("input") is None)


def _wb_members(case, seed):
  rng = np.random.default_rng(seed)
  out = []
  for m in case["members"]:
    m = m if isinstance(m, dict) else dict(dims=m)
    dims = m["dims"]
    ws = [orc.glorot_uniform(rng, dims[i], dims[i + 1]) for i in range(len(dims) - 1)]
    bs = [(rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32) for i in range(len(dims) - 1)]
    if m.get("image"):
      cin = m["image"][2]
      f = dims[0] // ((m["image"][0] // 2) * (m["image"][1] // 2))
      ws = [(rng.standard_normal((3, 3, cin, f)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)] + ws
      bs = [(rng.standard_normal(f) * 0.1).astype(np.float32)] + bs
    depth = len(dims) - 2 + (1 if m.get("image") else 0)
    out.append(dict(dims=dims, image=m.get("image"), ws=ws, bs=bs, cx=float(np.sqrt(np.float32(depth)))))
  return out


def _wb_weights(case, members, seed):
  rng = np.random.default_rng(seed + 1)
  N, C = len(members), case["C"]
  if case.get("mean"):
    w = np.zeros((N,), np.float32)
    w[case["mean"]:] = np.float32(1.0 / (N - case["mean"]))
  elif case["mix"] == "scalar":
    w = rng.uniform(0.2, 0.8, N).astype(np.float32)
  elif case["mix"] == "vector":
    w = rng.uniform(-0.5, 1.0, (N, C)).astype(np.float32)
  else:
    w = [(rng.standard_normal((m["dims"][-2], C)) * 0.2).astype(np.float32) for m in members]
  bias = (rng.standard_normal(C) * 0.1).astype(np.float32) if case.get("bias") else np.zeros((C,), np.float32)
  return w, bias


def _wb_batch(case, B, seed):
  rng = np.random.default_rng(seed)
  C = case["C"]
  x = rng.standard_normal((B, case.get("input", D))).astype(np.float32)
  if case["head"] == "softmax_xent":
    y = rng.integers(0, C, B).astype(np.int64)
  elif case["head"] == "mse":
    y = rng.standard_normal((B, C)).astype(np.float32)
  else:
    y = rng.integers(0, 2, (B, C)).astype(np.float32)
  return x, y


def wb_reference(case, members, w, bias, x, y, gammas, floor, fp32_dot):
  outs = [member64(m["ws"], m["bs"], x, m["image"], floor, fp32_dot) for m in members]
  if case["mix"] == "matrix":
    logits, errs = [], []
    for (_, _, last, lE), W in zip(outs, w):
      z, zb = layer_fwd(last, W, np.zeros(case["C"]), False)
      _, own = layer_fwd(np.abs(last) + lE, np.abs(f64(W)), np.zeros(case["C"]), False, floor=floor, fp32_dot=fp32_dot)
      logits.append(z)
      errs.append(own + lE @ np.abs(f64(W)))
  else:
    logits, errs = [o[0] for o in outs], [o[1] for o in outs]
  return ensemble64(case["head"], case["mix"], w, bias, logits, errs, y, gammas)


def check_members(fails, nets, params, x, rows, floor, fp32_dot, tag, mw=None, mw_logits=None):
  """Teacher-forced: every layer of every member (the conv stem's pooled features too) from the engine's own input to
  it, on the first `rows` examples, within one layer's bound -- the carried bound of a deep member is far too loose to
  see a wrong layer.  Returns the engine's member logits (MATRIX: its weighted last layers, checked the same way)."""
  from tests.test_gpu_step_state import _acts, _merge
  out = []
  for k, (net, (ws, bs, image)) in enumerate(zip(nets, params)):
    h = f64(x[:rows])
    what = "%s member %d" % (tag, k)
    if image is not None:
      st = conv_stem64(h.reshape((-1,) + tuple(image)), ws[0], bs[0])
      got = _merge(net.stem_out, net.batch, net.dims[0])[:rows]
      _check(fails, "member layers", got, st["pooled"], st["bound"] + floor, what + " conv stem")
      h, ws, bs = f64(got), ws[1:], bs[1:]
    acts = [a[:rows] for a in _acts(net, net.batch, not fp32_dot)]
    for i, (w, b) in enumerate(zip(ws, bs)):
      last = i == len(ws) - 1
      exact, bound = layer_fwd(h, w, b, not last, floor=floor, fp32_dot=fp32_dot)
      got = net.logits.cpu().numpy()[:rows] if last else acts[i]
      _check(fails, "member layers", got, exact, bound, "%s layer %d" % (what, i))
      if last and mw is not None:
        exact, bound = layer_fwd(h, mw[k], np.zeros(np.shape(mw[k])[1]), False, floor=floor)
        got = mw_logits[k].cpu().numpy()[:rows]
        _check(fails, "member layers", got, exact, bound, "%s last layer x W_%d" % (what, k))
      h = f64(got)
    out.append(h)
  return out


def _snapshot(nets):
  ts = []
  for n in nets:
    ts += n.ws + n.bs + (n.wps or []) + ([n.stem_k, n.stem_b] if n.stem else [])
  return [t.clone() for t in ts]


def _same_bytes(a, b):
  import torch
  return all(x.shape == y.shape and torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))


def check_forced(fails, case, plan, nets, members, w, bias, x, y, rows, gammas, floor, fp32_dot, tag, got3=None):
  """the members layer by layer, then the ensemble logits and out3 from the engine's member logits"""
  mat = case["mix"] == "matrix"
  ml = check_members(fails, nets, [(m["ws"], m["bs"], m["image"]) for m in members], x, rows, floor, fp32_dot, tag,
                     mw=w if mat else None, mw_logits=plan.mw_logits if mat else None)
  e, e_err, out3, out3_b = ensemble64(case["head"], case["mix"], w, bias, ml, [0.0] * len(ml), y, gammas)
  _check(fails, "ensemble logits", plan.ens_logits[:rows].cpu().numpy(), e, e_err, tag + " ens_logits")
  got3 = plan.out3.cpu().numpy() if got3 is None else got3
  _check(fails, "ensemble out3", got3, out3, out3_b, tag + " out3")


def run_white_box(name, planes, f16):
  import torch
  from adanet_b200.core import engine as eng
  case = WB_CASES[name]
  B, C = case["B"], case["C"]
  members = _wb_members(case, 7)
  w, bias = _wb_weights(case, members, 7)
  lam, beta = case.get("reg", (0.0, 0.0))
  gammas = [gamma32(lam, beta, m["cx"]) if (lam or beta) else 0.0 for m in members]
  dev = torch.device("cuda", torch.cuda.current_device())
  nets = [eng.DenseNet("m%d" % k, m["dims"], m["ws"], m["bs"], m["cx"], B, dev, image_shape=m["image"])
          for k, m in enumerate(members)]
  ens = (eng.EnsemblerPlanSpec(optimizer=None, mixture_weight_type="scalar", kind="mean", name="mean") if case.get("mean")
         else eng.EnsemblerPlanSpec(mixture_weight_type=case["mix"], adanet_lambda=lam, adanet_beta=beta,
                                    use_bias=bool(case.get("bias"))))
  plan = eng.EnsembleEvalPlan(nets, w, bias, ens, case["head"], B, C, dev)
  assert (plan.xp is not None) == planes
  floor = F16_FLOOR if f16 else 0.0
  snap = _snapshot(nets)
  fails = []
  x, y = _wb_batch(case, B, 11)
  got3 = np.asarray(plan.run(x, y))
  torch.cuda.synchronize()
  logits = plan.ens_logits.clone()
  check_forced(fails, case, plan, nets, members, w, bias, x, y, B, gammas, floor, not planes, name)
  e, e_err, out3, out3_b = wb_reference(case, members, w, bias, x, y, gammas, floor, not planes)
  _check(fails, "carried: logits", logits.cpu().numpy(), e, e_err, "%s ens_logits (carried bound)" % name)
  _check(fails, "carried: out3", got3, out3, out3_b, "%s out3 (carried bound)" % name)
  if not np.array_equal(plan.out3.cpu().numpy(), got3.astype(np.float32)):
    fails.append("%s: run() returned %s, out3 holds %s" % (name, got3, plan.out3.cpu().numpy()))
  # the same call again: the same bytes; without labels (predict): the same logits
  again = np.asarray(plan.run(x, y))
  if not (np.array_equal(again, got3) and _same_bytes([plan.ens_logits], [logits])):
    fails.append("%s: a second run differs" % name)
  plan.run(x, None)
  if not _same_bytes([plan.ens_logits], [logits]):
    fails.append("%s: run(x, None) gives other logits" % name)
  # a partial batch: the first b rows of the static buffers
  b = max(1, B // 2 - 1)
  xb, yb = _wb_batch(case, b, 12)
  got3 = np.asarray(plan.run(xb, yb))
  if plan.rows != b:
    fails.append("%s: rows %d after a batch of %d" % (name, plan.rows, b))
  check_forced(fails, case, plan, nets, members, w, bias, xb, yb, b, gammas, floor, not planes, "%s, %d rows" % (name, b),
               got3)
  e, e_err, out3, out3_b = wb_reference(case, members, w, bias, xb, yb, gammas, floor, not planes)
  _check(fails, "carried: logits", plan.ens_logits[:b].cpu().numpy(), e, e_err, "%s ens_logits of %d rows" % (name, b))
  _check(fails, "carried: out3", got3, out3, out3_b, "%s out3 of %d rows" % (name, b))
  torch.cuda.synchronize()
  if not _same_bytes(_snapshot(nets), snap):
    fails.append("%s: run() changed a member's weights or planes" % name)
  assert not fails, "\n".join(fails[:30])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(WB_CASES))
def test_eval_plan_white_box(fmt, name):
  from adanet_b200 import _lib
  run_white_box(name, True, _lib.plane_format() == _lib.PLANES_F16)


def _dense_path(_lib):
  """the dense path in force (adn_set_dense_path / ADN_DENSE_PATH), read back through the path the library picks for
  a shape the tensor path supports and for one it does not: SIMT everywhere, -1 (refused) when the tensor path is
  forced, SIMT only for the small shape under AUTO"""
  if _lib.query(_lib.Q_DENSE_FWD_PATH, 1 << 20, 1024, 1024) == _lib.PATH_SIMT:
    return _lib.PATH_SIMT
  return _lib.PATH_AUTO if _lib.query(_lib.Q_DENSE_FWD_PATH, 1, 1, 1) == _lib.PATH_SIMT else _lib.PATH_TCGEN05


@pytest.fixture
def simt():
  torch, _lib, lib = _open()
  before = _dense_path(_lib)
  _lib.set_dense_path(_lib.PATH_SIMT)
  _PATH[0] = "simt"
  try:
    yield
  finally:
    _lib.set_dense_path(before)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SIMT_WB)
def test_eval_plan_white_box_simt(simt, name):
  run_white_box(name, False, False)


# ------------------------------------------------------------------------------------------------------------------
# IterationPlan.eval_step after two training steps
# ------------------------------------------------------------------------------------------------------------------
EVAL_STEP_CASES = ["dropout", "vector_warm", "matrix", "mse", "sigmoid", "shared", "cnn"]


def _net_params(plan, fnets, frozen, st, net):
  """(ws, bs, image) of a net of the plan: frozen members from the case, candidates from the state dict"""
  for f, fs in zip(fnets, frozen):
    if f is net:
      return fs["p"][0], fs["p"][1], None
  c = next(c for c in plan.candidates if c.net is net)
  key = "c%d_" % c.index
  ws = [st[key + "w%d" % i] for i in range(len(c.net.ws))]
  bs = [st[key + "b%d" % i] for i in range(len(c.net.bs))]
  if c.net.stem:
    return [st[key + "stem_k"]] + ws, [st[key + "stem_b"]] + bs, c.net.image_shape
  return ws, bs, None


def _head_setup(case, plan, fnets, frozen, st, gidx, h):
  """(member nets, their params, mix, w, bias, gammas) of candidate ensemble `gidx`, from the case and the state"""
  from adanet_b200 import _lib
  from tests.test_gpu_step_state import _head_key
  nets = _members(case, plan, fnets, gidx, h)
  key = _head_key(plan, gidx, h)
  N = len(nets)
  if h.kind == "mean":
    # mean.py:92-135: the candidate's new subnetworks averaged, previous members ignored
    w = np.zeros((N,), np.float32)
    w[h.n_prev:] = np.float32(1.0 / (N - h.n_prev))
    mix, gam = "scalar", [0.0] * N
  else:
    mix = {_lib.MIX_SCALAR: "scalar", _lib.MIX_VECTOR: "vector", _lib.MIX_MATRIX: "matrix"}[h.mix]
    w = [st[key + "mix%d" % k] for k in range(N)] if mix == "matrix" else st[key + "mix0"]
    gam = [gamma32(h.ens.adanet_lambda, h.ens.adanet_beta, n.complexity) if (h.ens.adanet_lambda or h.ens.adanet_beta)
           else 0.0 for n in nets]
  members = [dict(zip(("ws", "bs", "image"), _net_params(plan, fnets, frozen, st, n))) for n in nets]
  return nets, members, mix, w, st[key + "bias"], gam


@pytest.mark.gpu
@pytest.mark.parametrize("name", EVAL_STEP_CASES)
def test_eval_step_metrics(fmt, name):
  """Every metric of every candidate ensemble after two training steps, on a full and on a partial hold-out batch,
  against float64 from the trained state; the training state byte-identical afterwards.  The dropout case's
  candidates must evaluate without their masks."""
  import torch
  from adanet_b200 import _lib
  from tests.test_gpu_step_state import _batch
  case = dict(CASES[name], inject=None)
  frozen, cands, warm = _case_data(case, seed=21)
  plan, fnets = _build_plan(case, frozen, cands, warm)
  for k in range(2):
    x, y = _batch(case, k)
    own = {c.index: _batch(case, 500 + k) for c in plan.candidates if c.bagged}
    plan.train_step(x, y, own_batches=own or None)
  before = plan.state_dict()
  f16 = _lib.plane_format() == _lib.PLANES_F16
  floor = F16_FLOOR if f16 else 0.0
  fails = []
  metrics = ["adanet_loss", "loss", "average_loss"] + ([] if case["head"] == "mse" else ["accuracy"])
  for rows in (case["B"], case["B"] // 2 + 1):
    xe, ye = _batch(case, 99)
    xe, ye = xe[:rows], ye[:rows]
    got = {m: plan.eval_step(xe, ye, m) for m in metrics}
    for j, (gidx, h, _) in enumerate(plan.heads):
      nets, members, mix, w, bias, gam = _head_setup(case, plan, fnets, frozen, before, gidx, h)
      tag = "%s %s, %d rows" % (name, h.name, rows)
      # the members as the last eval_step left them (no dropout), the metrics from their logits
      ml = check_members(fails, nets, [(m["ws"], m["bs"], m["image"]) for m in members], xe, rows, floor, False, tag,
                         mw=w if mix == "matrix" else None, mw_logits=h.mw_logits if mix == "matrix" else None)
      e, e_err, out3, out3_b = ensemble64(case["head"], mix, w, bias, ml, [0.0] * len(ml), ye, gam)
      _check(fails, "eval_step adanet_loss", got["adanet_loss"][j], out3[2], out3_b[2], tag + " adanet_loss")
      for m in ("loss", "average_loss"):
        _check(fails, "eval_step loss", got[m][j], out3[0], out3_b[0], "%s %s" % (tag, m))
      if "accuracy" in got:
        check_accuracy(fails, case["head"], got["accuracy"][j], e, e_err, ye, tag)
      _, _, c3, c3_b = wb_reference(dict(C=case["C"], head=case["head"], mix=mix), members, w, bias, xe, ye, gam, floor,
                                    False)
      _check(fails, "carried: out3", got["adanet_loss"][j], c3[2], c3_b[2], tag + " adanet_loss (carried bound)")
  after = plan.state_dict()
  for key in before:
    if not np.array_equal(before[key], after[key], equal_nan=True):
      fails.append("eval_step changed %s" % key)
  torch.cuda.synchronize()
  assert not fails, "\n".join(fails[:30])


# ------------------------------------------------------------------------------------------------------------------
# Estimator: evaluate / predict over a ragged tail, a fresh Estimator, the Evaluator
# ------------------------------------------------------------------------------------------------------------------
EB, ED = 64, 20


def _est_data(kind, n, seed):
  rng = np.random.default_rng(seed)
  if kind == "cnn":
    x = (rng.uniform(0, 1, (n, 8, 8, 3)) * 2 - 1).astype(np.float32)
    return x, rng.integers(0, 4, n).astype(np.int64)
  x = rng.standard_normal((n, ED)).astype(np.float32)
  t = x @ np.random.default_rng(5).standard_normal((ED, 4)).astype(np.float32)
  if kind == "softmax":
    return x, t.argmax(axis=1).astype(np.int64)
  if kind == "sigmoid":
    return x, (t[:, :1] > 0).astype(np.float32)
  return x, (t[:, :3] * 0.5).astype(np.float32)


def _input_fn(x, y, key, batch=EB):
  def fn():
    for i in range(0, x.shape[0], batch):
      yield {key: x[i:i + batch]}, y[i:i + batch]
  return fn


def _make_estimator(kind, model_dir, evaluator=None, steps=4):
  import adanet_b200 as adanet
  from adanet_b200 import graph, train
  from adanet_b200.examples import simple_cnn, simple_dnn
  head = {"softmax": adanet.heads.MultiClassHead(4), "sigmoid": adanet.heads.BinaryClassHead(),
          "mse": adanet.heads.RegressionHead(3), "cnn": adanet.heads.MultiClassHead(4)}[kind]
  if kind == "cnn":
    gen = simple_cnn.SimpleCNNGenerator(0.01, steps, seed=3, num_candidates=2)
    ensemblers = None
  else:
    gen = simple_dnn.Generator(feature_columns=[graph.numeric_column("x", ED)], optimizer=train.GradientDescentOptimizer(0.05),
                               layer_size=16, learn_mixture_weights=True, seed=7)
    mix = {"softmax": dict(), "sigmoid": dict(mixture_weight_type="vector", use_bias=True),
           "mse": dict(mixture_weight_type="matrix")}[kind]
    ensemblers = [adanet.ensemble.ComplexityRegularizedEnsembler(optimizer=train.GradientDescentOptimizer(0.05),
                                                                 adanet_lambda=0.01, adanet_beta=0.002, **mix)]
  return adanet.Estimator(head=head, subnetwork_generator=gen, max_iteration_steps=steps, ensemblers=ensemblers,
                          max_iterations=2, model_dir=model_dir, evaluator=evaluator)


def _saved_ensemble(model_dir, kind):
  """the members, mixture weights and bias of ensemble-latest.npz / .json, and the ensembler's (mix, lambda, beta)"""
  with np.load(os.path.join(model_dir, "ensemble-latest.npz")) as npz:
    data = dict(npz)
  with open(os.path.join(model_dir, "ensemble-latest.json")) as f:
    meta = json.load(f)
  members = []
  for k, m in enumerate(meta["members"]):
    n = len(m["dims"]) - 1 + (1 if m.get("image_shape") else 0)
    members.append(dict(ws=[data["m%d_w%d" % (k, i)] for i in range(n)], bs=[data["m%d_b%d" % (k, i)] for i in range(n)],
                        image=m.get("image_shape"), cx=m["complexity"], dims=m["dims"]))
  mix, lam, beta = {"softmax": ("scalar", 0.01, 0.002), "sigmoid": ("vector", 0.01, 0.002), "mse": ("matrix", 0.01, 0.002),
                    "cnn": ("scalar", 0.0, 0.0)}[kind]
  w = [data["mixture_weight_%d" % k] for k in range(len(members))] if mix == "matrix" else data["mixture_weights"]
  return members, w, data["bias"], mix, lam, beta


HEAD_OF = {"softmax": "softmax_xent", "sigmoid": "sigmoid_xent", "mse": "mse", "cnn": "softmax_xent"}


def _est_reference(model_dir, kind, x, y, f16):
  members, w, bias, mix, lam, beta = _saved_ensemble(model_dir, kind)
  gam = [gamma32(lam, beta, m["cx"]) if (lam or beta) else 0.0 for m in members]
  xf = x.reshape(x.shape[0], -1)
  case = dict(C=np.size(bias), head=HEAD_OF[kind], mix=mix)
  return wb_reference(case, members, w, bias, xf, y, gam, F16_FLOOR if f16 else 0.0, False)


def check_evaluate_predict(fails, est, kind, model_dir, xe, ye, f16, tag):
  """evaluate over an input with a ragged tail (the reference's two weightings), predict one row per example"""
  import torch
  key = "images" if kind == "cnn" else "x"
  head = HEAD_OF[kind]
  ev = est.evaluate(_input_fn(xe, ye, key))
  losses, bounds, sizes = [], [], []
  for i in range(0, xe.shape[0], EB):
    _, _, out3, out3_b = _est_reference(model_dir, kind, xe[i:i + EB], ye[i:i + EB], f16)
    losses.append(out3[0])
    bounds.append(out3_b[0])
    sizes.append(min(EB, xe.shape[0] - i))
  sz = np.asarray(sizes, dtype=np.float64)
  _check(fails, "evaluate loss", ev["loss"], np.mean(losses), np.mean(bounds) + 4 * U * abs(np.mean(losses)), tag + " loss")
  avg = (sz * losses).sum() / sz.sum()
  _check(fails, "evaluate loss", ev["average_loss"], avg, (sz * bounds).sum() / sz.sum() + 4 * U * abs(avg),
         tag + " average_loss")
  e, e_err, _, _ = _est_reference(model_dir, kind, xe, None, f16)
  if head == "mse":
    if "accuracy" in ev:
      fails.append("%s: a regression head reports accuracy" % tag)
  elif "accuracy" not in ev:
    fails.append("%s: evaluate reports no accuracy" % tag)
  else:
    check_accuracy(fails, head, ev["accuracy"], e, e_err, ye, tag + " evaluate")
  preds = list(est.predict(_input_fn(xe, ye, key)))
  if len(preds) != xe.shape[0]:
    fails.append("%s: predict yielded %d rows for %d examples" % (tag, len(preds), xe.shape[0]))
    return None
  logits = np.stack([p["logits"] for p in preds])
  _check(fails, "predict logits", logits, e, e_err, tag + " logits")
  l64 = f64(logits)
  if head == "softmax_xent":
    z = np.exp(l64 - l64.max(axis=1, keepdims=True))
    p = z / z.sum(axis=1, keepdims=True)
    got = np.stack([q["probabilities"] for q in preds])
    _check(fails, "predict probabilities", got, p, 8 * U * p + 1e-30, tag + " probabilities")
    ids = np.stack([q["class_ids"] for q in preds]).reshape(-1)
    if not np.array_equal(ids, logits.argmax(axis=1)):
      fails.append("%s: class_ids are not the arg-max of the logits" % tag)
    amb = ambiguous(head, e, e_err)
    if not np.array_equal(ids[~amb], e.argmax(axis=1)[~amb]):
      fails.append("%s: class_ids differ from float64 where the top-2 margin is clear" % tag)
  elif head == "sigmoid_xent":
    got = np.stack([q["logistic"] for q in preds])
    s = 1.0 / (1.0 + np.exp(-l64))
    _check(fails, "predict logistic", got, s, 4 * U * s + 1e-30, tag + " logistic")
  else:
    got = np.stack([q["predictions"] for q in preds])
    if not np.array_equal(got, logits):
      fails.append("%s: predictions are not the logits" % tag)
  return logits


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["softmax", "sigmoid", "mse", "cnn"])
def test_estimator_evaluate_predict_ragged_tail(fmt, kind, tmp_path):
  """Two iterations, then evaluate / predict over 2.5 batches against float64 of ensemble-latest.npz; a fresh
  Estimator on the same model_dir predicts the same bytes."""
  from adanet_b200 import _lib
  f16 = _lib.plane_format() == _lib.PLANES_F16
  key = "images" if kind == "cnn" else "x"
  x, y = _est_data(kind, EB * 8, 1)
  est = _make_estimator(kind, str(tmp_path))
  est.train(_input_fn(x, y, key), max_steps=8)
  assert est._search.iteration == 2
  xe, ye = _est_data(kind, EB * 2 + EB // 2, 2)
  fails = []
  logits = check_evaluate_predict(fails, est, kind, str(tmp_path), xe, ye, f16, "%s %s" % (fmt, kind))
  assert not fails, "\n".join(fails[:30])
  fresh = _make_estimator(kind, str(tmp_path))
  again = np.stack([p["logits"] for p in fresh.predict(_input_fn(xe, ye, key))])
  assert again.tobytes() == logits.tobytes(), "a fresh Estimator on the same model_dir predicts other logits"


def _spy(monkeypatch):
  """records, at each Evaluator pass, what the ranked values are computed from: every candidate ensemble's trained
  state (IterationPlan.eval_step) and the previous ensemble (EnsembleEvalPlan.metric)"""
  from adanet_b200.core import engine as eng
  seen = dict(cands=[], prev=[])
  step, metric = eng.IterationPlan.eval_step, eng.EnsembleEvalPlan.metric

  def eval_step(self, x, y, m="adanet_loss"):
    if not seen["cands"] or seen["cands"][-1][0] is not self:
      members = [[(f.numpy_params(), f.image_shape if f.stem else None, f.complexity) for f in h.member_nets]
                 for _, h, _ in self.heads]
      seen["cands"].append((self, self.state_dict(), members))
    return step(self, x, y, m)

  def prev_metric(self, x, y, m="adanet_loss"):
    if not seen["prev"] or seen["prev"][-1][0] is not self:
      seen["prev"].append((self, [(n.numpy_params(), n.image_shape if n.stem else None, n.complexity) for n in self.members],
                           self.mix_w.cpu().numpy(), self.bias.cpu().numpy(), list(self.gammas)))
    return metric(self, x, y, m)

  monkeypatch.setattr(eng.IterationPlan, "eval_step", eval_step)
  monkeypatch.setattr(eng.EnsembleEvalPlan, "metric", prev_metric)
  return seen


def _ranked64(metric, head, members, w, bias, gam, xh, yh, f16):
  """(value, bound) of an Evaluator metric over the hold-out batches: adanet_loss per batch, accuracy per example"""
  ms = [dict(ws=p[0], bs=p[1], image=img) for p, img, _ in members]
  case = dict(C=np.size(bias), head=head, mix="scalar")
  vals, bds, es = [], [], []
  for i in range(0, xh.shape[0], EB):
    e, e_err, out3, out3_b = wb_reference(case, ms, w, bias, xh[i:i + EB], yh[i:i + EB], gam, F16_FLOOR if f16 else 0.0,
                                          False)
    vals.append(out3[2])
    bds.append(out3_b[2])
    es.append((e, e_err))
  if metric == "adanet_loss":
    return np.mean(vals), np.mean(bds) + 4 * U * abs(np.mean(vals)), None
  return None, None, (np.concatenate([a for a, _ in es]), np.concatenate([b for _, b in es]))


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["adanet_loss", "accuracy"])
def test_evaluator_ragged_holdout(fmt, metric, monkeypatch):
  """An Evaluator whose hold-out input ends in a partial batch: every candidate's ranked value at both iterations,
  and the previous ensemble's at iteration 1, against float64 of the state they were computed from."""
  import adanet_b200 as adanet
  from adanet_b200 import _lib
  f16 = _lib.plane_format() == _lib.PLANES_F16
  seen = _spy(monkeypatch)
  x, y = _est_data("softmax", EB * 8, 1)
  xh, yh = _est_data("softmax", EB * 2 + 24, 3)
  ev = adanet.Evaluator(input_fn=_input_fn(xh, yh, "x"), metric_name=metric,
                        objective="minimize" if metric == "adanet_loss" else "maximize")
  est = _make_estimator("softmax", None, evaluator=ev)
  est.train(_input_fn(x, y, "x"), max_steps=8)
  reps = est._search.reports
  assert len(reps) == 2 and len(seen["cands"]) == 2 and len(seen["prev"]) == 1
  fails = []
  for t, (rep, (plan, st, members)) in enumerate(zip(reps, seen["cands"])):
    got = rep.ema_losses[1:] if t else rep.ema_losses
    for j, (_, h, _) in enumerate(plan.heads):
      key = "c%d_" % next(c.index for c in plan.candidates if c.ehead is h)
      gam = [gamma32(0.01, 0.002, cx) for _, _, cx in members[j]]
      v, b, eb = _ranked64(metric, "softmax_xent", members[j], st[key + "mix0"], st[key + "bias"], gam, xh, yh, f16)
      tag = "iteration %d %s" % (t, h.name)
      if metric == "adanet_loss":
        _check(fails, "evaluator adanet_loss", got[j], v, b, tag)
      else:
        check_accuracy(fails, "softmax_xent", got[j], eb[0], eb[1], yh, tag)
  _, members, w, bias, gam = seen["prev"][0]
  assert gam == [gamma32(0.01, 0.002, cx) for _, _, cx in members]
  v, b, eb = _ranked64(metric, "softmax_xent", members, w, bias, gam, xh, yh, f16)
  if metric == "adanet_loss":
    _check(fails, "evaluator adanet_loss", reps[1].ema_losses[0], v, b, "iteration 1 previous_ensemble")
  else:
    check_accuracy(fails, "softmax_xent", reps[1].ema_losses[0], eb[0], eb[1], yh, "iteration 1 previous_ensemble")
  assert not fails, "\n".join(fails[:30])


# ------------------------------------------------------------------------------------------------------------------
# the fp16 -> TF32 fallback
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["softmax", "mse"])
def test_eval_plan_follows_a_plane_format_switch(kind, tmp_path):
  """The eval plan is built under fp16 planes; after a switch to TF32 planes (what the fallback after an fp16
  overflow does mid-training) the plan the Estimator hands out must have buffers of the TF32 size -- checked before
  anything is launched -- and evaluate correctly."""
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _lib.set_plane_format(_lib.PLANES_F16)
  try:
    _PATH[0] = "f16 -> tf32"
    x, y = _est_data(kind, EB * 8, 1)
    est = _make_estimator(kind, str(tmp_path))
    est.train(_input_fn(x, y, "x"), max_steps=8)
    plan16 = est._ensemble_eval_plan()
    _lib.set_plane_format(_lib.PLANES_TF32)
    plan = est._ensemble_eval_plan()
    size = lambda r, c: _lib.query(_lib.Q_PLANES_BYTES, r, c)
    assert plan.xp.numel() * 4 == size(plan.batch, plan.x.shape[1]), "the eval plan's input planes keep the fp16 size"
    assert (plan.mix == _lib.MIX_MATRIX) == (kind == "mse")
    if plan.mix == _lib.MIX_MATRIX:
      assert len(plan.mw) == len(plan.mwp) == len(plan.members)
      for W, wp in zip(plan.mw, plan.mwp):
        assert wp.numel() * 4 == size(W.shape[0], W.shape[1]), "the eval plan's MATRIX weight planes keep the fp16 size"
    for m in plan.members:
      for i, wp in enumerate(m.wps):
        assert wp.numel() * 4 == size(m.dims[i], m.dims[i + 1]), "member %s keeps fp16 weight planes" % m.name
      for i, hp in enumerate(m.hp):
        assert hp.numel() * 4 == size(m.batch, m.dims[i + 1]), "member %s keeps fp16 activation planes" % m.name
    assert plan is not plan16
    xe, ye = _est_data(kind, EB * 2 + 5, 2)
    fails = []
    check_evaluate_predict(fails, est, kind, str(tmp_path), xe, ye, False, "f16 -> tf32 " + kind)
    assert not fails, "\n".join(fails[:30])
  finally:
    _lib.set_plane_format(before)
