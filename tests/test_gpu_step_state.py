"""Whole training steps of IterationPlan (core/engine.py: _enqueue_waves, CandidatePlan, EnsembleHead), element by
element against a float64 restatement of one step (SURVEY.md section 3.3 steps 1-13) over an explicit state.

The per-step scalar losses that test_gpu_iteration / test_gpu_multi / test_gpu_api compare cannot see a wrong
gradient in a tensor that barely moves the loss, an optimizer slot that has not acted yet, or weight planes that no
longer equal split(W).  Here every step is teacher-forced: the state is read with IterationPlan.state_dict() before
the step, and each stage of the step is compared with float64 fed the engine's own values from the stage before, so
one step's rounding never decides the next one's tolerance:

  forward   every hidden layer (merged from its planes) = relu(h_{i-1} W_i + b_i) [* keep / (1 - rate)] from the
            engine's h_{i-1}; sign bits = the stored values; K padding zero; logits; the frozen members too
  heads     sub_out3 / dlogits / the logits layer's db; every ensemble head's out3, d_mix_w, d_bias
  backward  every dW_i, db_i against a chain from the engine's dlogits with masks from the engine's h; the chain
            carries a componentwise error bound, so a ReLU kink never makes the test flaky
  update    the TF1 rule applied in float64 to the engine's gradients and pre-step state: parameters and slots
            within a few fp32 ulps, step counters exact, weight planes byte-identical to a fresh split of the new
            weights, the EMA, the trace row at step_dev % capacity and step_dev + 1
  frozen    members' parameters and planes byte-identical across the step

Step 1 runs eagerly, step 2 captures the CUDA graph and replays it, step 3 replays.  Cases that inject a state with
load_state_dict inject it again before step 3, into the tensors the captured graph reads.

Bounds are componentwise: TOL (|A| |B|) plus the bias term.  fp16 planes carry 22 significant bits only above 2^-14;
below, a stored value is off by up to 2^-36 in scaled units (csrc/plane_fmt.cuh).  That absolute floor, derived from
the tensor's scale exponent, is added to the bound instead of loosening TOL; the small gradients of deep layers live
there.  The worst err/bound of every stage and the share of the deep nets' dW bound that is floor are printed at the
end of the module (pytest -s).
"""

import math
import os
import socket

import numpy as np
import pytest

from tests.parity_util import orc
from tests.test_gpu_plane_groups import _cw

TOL = 3e-6                  # one GEMM entry / one reduction, as in test_gpu_plane_groups
U = 2.0 ** -24              # fp32 unit roundoff
TOLH = 2e-6                 # the heads: exp / log / a C-term sum per entry
FLT_MIN = 2.0 ** -126       # a probability below fp32's normal range may underflow to 0
F16_FLOOR = 2.0 ** -36      # absolute error of an fp16 plane pair below 2^-14, in scaled units

# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
D = 100
ENS = dict(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001)


def _cands_mixed(C):
  return [dict(dims=[D, 96, 40, C], opt=("sgd", 0.05)),
          dict(dims=[D, 40, 130, 72, C], opt=("momentum", 0.02, 0.9)),
          dict(dims=[D, C], opt=("rmsprop", 0.01)),
          dict(dims=[D] + [24] * 8 + [C], opt=("adam", 0.01), deep=True)]


def _inject_opt_state(plan, st, rng, k):
  """Adam at step 10^5, RMSProp ms != 1 with a momentum slot, nonzero Momentum accumulators, momentum_cosine before, at
  and after decay_steps (DECAY)"""
  for c in plan.candidates:
    kind = c.spec.optimizer[0]
    pre = "c%d_sub_opt_" % c.index
    for key in [s for s in st if s.startswith(pre + "s0_") or s.startswith(pre + "s1_")]:
      shape = st[key].shape
      if kind == "rmsprop" and "_s0_" in key:
        st[key] = rng.uniform(0.05, 2.0, shape).astype(np.float32)          # ms > 0
      elif kind == "adam" and "_s1_" in key:
        st[key] = (rng.uniform(0.0, 1e-3, shape) ** 2).astype(np.float32)   # v >= 0, some tiny
      else:
        st[key] = (rng.standard_normal(shape) * 0.01).astype(np.float32)
    if kind == "adam":
      st[pre + "step"] = np.asarray(10 ** 5 + k, dtype=np.int64)
    if kind == "momentum_cosine":
      st[pre + "step"] = np.asarray(c.spec.optimizer[3] + (-1, 0, 5)[c.index % 3] + k, dtype=np.int64)


def _inject_step(value):
  def inject(plan, st, rng, k):
    st["step_dev"] = np.asarray(value + k, dtype=np.int64)
  return inject


DECAY = 20
CASES = {
    # two frozen members (one linear), narrowing / widening / linear / 8-deep candidates on the four TF1 optimizers
    "mixed": dict(B=256, C=10, head="softmax_xent", frozen=[[D, 48, 10], [D, 10]], cands=_cands_mixed(10), ens=ENS),
    # VECTOR mixture weights + bias, warm-started from the previous ensemble, Adam on the mixture weights
    "vector_warm": dict(B=256, C=10, head="softmax_xent", frozen=[[D, 32, 10], [D, 10]],
                        cands=[dict(dims=[D, 40, 130, 10], opt=("sgd", 0.05)), dict(dims=[D, 64, 10], opt=("adam", 0.01))],
                        ens=dict(optimizer=("adam", 0.01), mixture_weight_type="vector", use_bias=True, adanet_lambda=0.02,
                                 adanet_beta=0.003, warm_start_mixture_weights=True), warm=True),
    "vector_warm_legacy": dict(B=256, C=10, head="softmax_xent", frozen=[[D, 32, 10], [D, 10]],
                               cands=[dict(dims=[D, 40, 130, 10], opt=("sgd", 0.05)), dict(dims=[D, 64, 10], opt=("adam", 0.01))],
                               ens=dict(optimizer=("adam", 0.01), mixture_weight_type="vector", use_bias=True,
                                        adanet_lambda=0.02, adanet_beta=0.003, warm_start_mixture_weights=True,
                                        legacy_train_op=True), warm=True),
    "mse": dict(B=256, C=3, head="mse", frozen=[[D, 3]],
                cands=[dict(dims=[D, 40, 72, 3], opt=("momentum", 0.01, 0.9)), dict(dims=[D, 3], opt=("sgd", 0.02))],
                ens=dict(ENS, use_bias=True)),
    "sigmoid": dict(B=256, C=1, head="sigmoid_xent", frozen=[[D, 20, 1]],
                    cands=[dict(dims=[D, 40, 72, 1], opt=("rmsprop", 0.01)), dict(dims=[D, 1], opt=("adam", 0.01))],
                    ens=dict(ENS, mixture_weight_type="vector", use_bias=True)),
    # dropout on some hidden layers, step_dev past 2^32 (the mask hashes its low 32 bits)
    "dropout": dict(B=256, C=10, head="softmax_xent", frozen=[[D, 10]],
                    cands=[dict(dims=[D, 64, 48, 10], opt=("sgd", 0.05), dropout=[(0.25, 7), None]),
                           dict(dims=[D, 32, 40, 24, 10], opt=("momentum", 0.02, 0.9), dropout=[None, (0.5, 9), (0.1, 3)])],
                    ens=ENS, inject=_inject_step(2 ** 32 + 3)),
    "b37": dict(B=37, C=10, head="softmax_xent", frozen=[[D, 10]],
                cands=[dict(dims=[D, 96, 40, 10], opt=("sgd", 0.05)), dict(dims=[D] + [24] * 8 + [10], opt=("adam", 0.01), deep=True)],
                ens=ENS),
    # scale exponent 13 (the fp16 gradient planes carry dz * 2^13)
    "b4097": dict(B=4097, C=10, head="softmax_xent", frozen=[[D, 10]],
                  cands=[dict(dims=[D, 130, 72, 10], opt=("sgd", 0.05)), dict(dims=[D] + [24] * 8 + [10], opt=("adam", 0.01), deep=True)],
                  ens=ENS),
    "b4096_w1024": dict(B=4096, C=10, head="softmax_xent", frozen=[],
                        cands=[dict(dims=[D, 1024, 1024, 10], opt=("momentum", 0.01, 0.9))], ens=ENS),
    "opt_state": dict(B=256, C=10, head="softmax_xent", frozen=[[D, 10]],
                      cands=[dict(dims=[D, 64, 40, 10], opt=("adam", 0.01)), dict(dims=[D, 40, 10], opt=("rmsprop", 0.01, 0.9, 0.5)),
                             dict(dims=[D, 72, 10], opt=("momentum", 0.02, 0.9))] +
                            [dict(dims=[D, 40, 10], opt=("momentum_cosine", 0.05, 0.9, DECAY, 0.1)) for _ in range(3)],
                      ens=dict(ENS, optimizer=("momentum", 0.01, 0.9)), inject=_inject_opt_state),
    # MATRIX mixture weights + bias over a frozen linear member (its last layer is the minibatch's own planes) and a
    # frozen hidden one: the heads' own plane GEMMs (mw_logits, mw_l1, dens, d_mw)
    "matrix": dict(B=256, C=10, head="softmax_xent", frozen=[[D, 10], [D, 48, 10]],
                   cands=[dict(dims=[D, 40, 72, 10], opt=("sgd", 0.05)), dict(dims=[D, 10], opt=("momentum", 0.02, 0.9))],
                   ens=dict(optimizer=("sgd", 0.05), mixture_weight_type="matrix", use_bias=True, adanet_lambda=0.01,
                            adanet_beta=0.001)),
    # Grow / Solo / All heads over shared subnetworks, a second ensembler over the same candidate, the MeanEnsembler
    "shared": dict(B=256, C=10, head="softmax_xent", frozen=[[D, 32, 10]],
                   cands=[dict(dims=[D, 40, 72, 10], opt=("sgd", 0.05)), dict(dims=[D, 64, 10], opt=("adam", 0.01))],
                   ens=ENS, heads=[("n0_grow", [0], True, None), ("n1_grow", [1], True, None), ("n0_solo", [0], False, None),
                                   ("all", [0, 1], True, None), ("n0_grow", [0], True, "second"), ("all", [0, 1], True, "mean")],
                   ensemblers=dict(second=dict(optimizer=("momentum", 0.01, 0.9), mixture_weight_type="vector", use_bias=True,
                                               adanet_lambda=0.02, name="second"),
                                   mean=dict(kind="mean", name="mean"))),
    # a bagged subnetwork (its own minibatch, one step before the main pass) with dropout, beside a plain one
    "bagging": dict(B=256, C=10, head="softmax_xent", frozen=[[D, 10]],
                    cands=[dict(dims=[D, 48, 40, 10], opt=("sgd", 0.05), dropout=[(0.25, 5), None], own=True),
                           dict(dims=[D, 64, 10], opt=("momentum", 0.02, 0.9))], ens=dict(ENS, use_bias=True)),
    # a SimpleCNN candidate (conv3x3 + ReLU + maxpool 2 + dense) on 8x8x3 images: dpool -> adn_conv_stem_bwd
    "cnn": dict(B=128, C=10, head="softmax_xent", input=192, frozen=[[192, 10]],
                cands=[dict(dims=[256, 32, 10], image=(8, 8, 3), opt=("momentum_cosine", 0.05, 0.9, DECAY, 0.1)),
                       dict(dims=[192, 40, 10], opt=("sgd", 0.05))], ens=ENS),
}
GPU_CASES = sorted(CASES)
# what the fp32 SIMT cross-check path accepts (no MATRIX, shared heads, dropout, bagging or conv stems)
SIMT_CASES = ["b37", "b4096_w1024", "b4097", "mixed", "mse", "opt_state", "sigmoid", "vector_warm", "vector_warm_legacy"]


def _case_data(case, seed):
  """initial weights (glorot, random biases), frozen members, warm-start values"""
  rng = np.random.default_rng(seed)
  C = case["C"]

  def net(dims):
    ws = [orc.glorot_uniform(rng, dims[i], dims[i + 1]) for i in range(len(dims) - 1)]
    bs = [(rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32) for i in range(len(dims) - 1)]
    return ws, bs

  frozen = [dict(dims=dims, cx=float(np.sqrt(np.float32(len(dims) - 2))), p=net(dims)) for dims in case["frozen"]]
  cands = []
  for k, c in enumerate(case["cands"]):
    ws, bs = net(c["dims"])
    if c.get("image"):          # conv stem: he-scaled HWIO kernel [3, 3, Cin, F] in front of the dense stack
      cin, f = c["image"][2], c["dims"][0] // ((c["image"][0] // 2) * (c["image"][1] // 2))
      ws = [(rng.standard_normal((3, 3, cin, f)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)] + ws
      bs = [(rng.standard_normal(f) * 0.1).astype(np.float32)] + bs
    cands.append(dict(c, name="n%d" % k, cx=float(np.sqrt(np.float32(len(c["dims"]) - 2))), p=(ws, bs)))
  warm = None
  if case.get("warm"):
    nf = len(frozen)
    mt = case["ens"].get("mixture_weight_type", "scalar")
    warm = (rng.uniform(0.2, 0.8, (nf,) if mt == "scalar" else (nf, C)).astype(np.float32),
            (rng.standard_normal(C) * 0.1).astype(np.float32))
  return frozen, cands, warm


def _batch(case, k):
  rng = np.random.default_rng(1000 + 17 * k + case["B"])
  B, C = case["B"], case["C"]
  x = rng.standard_normal((B, case.get("input", D))).astype(np.float32)
  if case["head"] == "softmax_xent":
    y = rng.integers(0, C, B).astype(np.int64)
  elif case["head"] == "mse":
    y = rng.standard_normal((B, C)).astype(np.float32)
  else:
    y = rng.integers(0, 2, (B, C)).astype(np.float32)
  return x, y


# ------------------------------------------------------------------------------------------------------------------
# float64 restatement of one step
# ------------------------------------------------------------------------------------------------------------------
def f64(a):
  return np.asarray(a, dtype=np.float64)


def _tol(k, fp32_dot):
  """TOL, or on the fp32 SIMT path the classical bound of a K-term fp32 dot product, (K + 2) U"""
  return max(TOL, (k + 2) * U) if fp32_dot else TOL


def layer_fwd(h, w, b, relu, keep=None, rate=0.0, floor=0.0, fp32_dot=False):
  """(exact, bound) of relu(h w + b) [* keep / (1 - rate)]; `floor` = absolute error of a plane entry below 2^-14"""
  h, w, b = f64(h), f64(w), f64(b)
  z = h @ w + b
  bound = _tol(h.shape[1], fp32_dot) * (np.abs(h) @ np.abs(w) + np.abs(b))
  if floor:
    bound += floor * (np.abs(w).sum(axis=0)[None, :] + np.abs(h).sum(axis=1)[:, None] + 1.0)
  if relu:
    z = np.maximum(z, 0.0)
  if keep is not None:
    z = np.where(keep, z / (1.0 - rate), 0.0)
    bound = bound / (1.0 - rate)
  return z, bound


def head_loss(kind, logits, y, e_err=None):
  """float64 (loss, loss bound, dloss/dlogits, its bound) of a mean-reduced head; e_err: componentwise error of the
  logits (an ensemble's logits are computed from the members' in fp32)"""
  l = f64(logits)
  B, C = l.shape
  e_err = np.zeros_like(l) if e_err is None else e_err
  emax = e_err.max(axis=1, keepdims=True)
  if kind == "softmax_xent":
    yi = np.asarray(y).reshape(-1)
    z = l - l.max(axis=1, keepdims=True)
    p = np.exp(z) / np.exp(z).sum(axis=1, keepdims=True)
    one = np.zeros_like(l)
    one[np.arange(B), yi] = 1.0
    per = -np.log(p[np.arange(B), yi])
    loss = per.mean()
    g = (p - one) / B
    # z = l - max is rounded in fp32 (|dz| <= U |z|), and exp turns that into a relative error of p: far-apart logits
    gb = (TOLH + 2 * U * np.abs(z)) * p / B + TOLH * one / B + 2.0 * p * emax / B
    lb = TOLH * (np.abs(per) + np.abs(l).max(axis=1)).mean() + 2.0 * emax.mean()
  elif kind == "mse":
    d = l - f64(y).reshape(l.shape)
    n = d.size
    loss = (d * d).sum() / n
    g = 2.0 * d / n
    gb = TOLH * 2.0 * (np.abs(l) + np.abs(f64(y).reshape(l.shape))) / n + 2.0 * e_err / n
    lb = TOLH * (d * d + np.abs(l) * np.abs(d)).sum() / n + (2.0 * np.abs(d) * e_err).sum() / n
  else:
    zt = f64(y).reshape(l.shape)
    per = np.maximum(l, 0) - l * zt + np.log1p(np.exp(-np.abs(l)))
    n = l.size
    loss = per.sum() / n
    sig = 1.0 / (1.0 + np.exp(-l))
    g = (sig - zt) / n
    gb = TOLH * (sig + zt) / n + 0.25 * e_err / n
    lb = TOLH * (np.abs(per) + np.abs(l)).sum() / n + (np.abs(sig - zt) * e_err).sum() / n
  return loss, lb, g, gb + FLT_MIN


def ensemble(kind, mix, mw, bias, members, y, gammas, reg_mult, use_bias):
  """steps 6-11 over the members' logits: ensemble logits, (loss, reg, adanet_loss), mixture-weight / bias gradients,
  each with its bound"""
  mw, bias = f64(mw), f64(bias)
  ms = [f64(m) for m in members]
  wk = [mw[k] for k in range(len(ms))]         # SCALAR: [] ; VECTOR: [C]
  e = bias + sum(w * m for w, m in zip(wk, ms))
  e_err = 2 * (len(ms) + 1) * U * (np.abs(bias) + sum(np.abs(w * m) for w, m in zip(wk, ms)))
  loss, lb, g, gb = head_loss(kind, e, y, e_err)
  reg_on = any(gm != 0.0 for gm in gammas)
  reg = sum(gm * np.abs(w).sum() for gm, w in zip(gammas, wk)) if reg_on else 0.0
  reg_b = 2 * (mw.size + len(ms)) * U * sum(gm * np.abs(w).sum() for gm, w in zip(gammas, wk)) if reg_on else 0.0
  axis = None if mix == "scalar" else 0
  dmw = np.stack([(g * m).sum(axis=axis) for m in ms])
  dmw_b = np.stack([TOL * (np.abs(g) * np.abs(m)).sum(axis=axis) + (gb * np.abs(m)).sum(axis=axis) for m in ms])
  if reg_on:
    dmw = dmw + np.stack([reg_mult * gm * np.sign(w) for gm, w in zip(gammas, wk)])
    dmw_b = dmw_b + np.stack([4 * U * reg_mult * gm * np.abs(np.sign(w)) for gm, w in zip(gammas, wk)])
  db = g.sum(axis=0) if use_bias else None
  db_b = (TOL * np.abs(g).sum(axis=0) + gb.sum(axis=0)) if use_bias else None
  out3 = np.array([loss, reg, loss + reg])
  out3_b = np.array([lb, reg_b, lb + reg_b]) + 4 * U * np.abs(out3)
  return dict(e=e, out3=out3, out3_b=out3_b, dmw=dmw, dmw_b=dmw_b, db=db, db_b=db_b, g=g)


def backward(ws, hs, dlogits, masks, dx_muls, floor=0.0, floor_x=0.0, tol=TOL, fp32_dot=False, h_err=None, amb=None,
             dz_err=None, dx0=False):
  """dW_i, db_i (i < n - 1: db of the logits layer comes from the head) and their bounds, from the engine's dlogits.
  hs[i] = input of layer i (hs[0] = x); masks[i] = hs[i] > 0 for i >= 1; dx_muls[i] multiplies the gradient w.r.t.
  hs[i].  The carried bound: E_i = (TOL (|dZ_{i+1}| |W^T|) + E_{i+1} |W^T| + floor terms) * m * dx_mul.
  `floor` = absolute error of a gradient plane entry (2^-36 / 2^s), `floor_x` of an activation plane entry; with
  tol = 0 the bounds are the floors' share alone.  fp32_dot: the fp32 SIMT path, TOL -> (K + 2) U.
  For a forward that is not the engine's own (the bagged pre-pass, whose activations the main pass overwrites):
  h_err[i] bounds the error of hs[i], amb[i] marks the entries whose ReLU / dropout mask the engine may have drawn
  either way, and dz_err bounds the error of dlogits.  dx0: the first layer also produces dX (below a conv stem,
  masked by masks[0]), returned as dx / dx_b."""
  n = len(ws)
  dz = f64(dlogits)
  B = dz.shape[0]
  err = tol * np.abs(dz) + floor + (dz_err if dz_err is not None else 0.0)   # the planes of dlogits: one rounding
  dws, dws_b, dbs, dbs_b = [None] * n, [None] * n, [None] * n, [None] * n
  out = {}
  for i in range(n - 1, -1, -1):
    h = f64(hs[i])
    dws[i] = h.T @ dz
    base = _tol(B, fp32_dot) * (np.abs(h).T @ np.abs(dz)) if tol else 0.0
    carried = np.abs(h).T @ err
    if h_err is not None and h_err[i] is not None:
      carried = carried + h_err[i].T @ (np.abs(dz) + err)
    fl = floor_x * np.abs(dz).sum(axis=0)[None, :] if floor_x else 0.0
    dws_b[i] = base + carried + fl
    if i == 0 and not dx0:
      break
    w = np.abs(f64(ws[i]))
    m = masks[i].astype(np.float64) * dx_muls[i]
    nz = (f64(dz) @ f64(ws[i]).T) * m
    full = _tol(dz.shape[1], fp32_dot) * (np.abs(dz) @ w.T) if tol else 0.0
    e = (full + err @ w.T) * m
    if floor:
      e += (floor * w.sum(axis=1)[None, :] + floor_x * np.abs(dz).sum(axis=1)[:, None]) * m + floor * (m != 0)
    if amb is not None and amb[i] is not None:
      e = e + amb[i] * dx_muls[i] * ((np.abs(dz) + err) @ w.T)
    if i == 0:
      out.update(dx=nz, dx_b=e)
      break
    dbs[i - 1] = nz.sum(axis=0)
    dbs_b[i - 1] = (_tol(B, fp32_dot) if tol else 0.0) * np.abs(nz).sum(axis=0) + e.sum(axis=0)
    dz, err = nz, e
  out.update(dw=dws, dw_b=dws_b, db=dbs, db_b=dbs_b)
  return out


def _fresh_slots(kind, p):
  """the slots an optimizer starts from (TF1: RMSProp's ms at 1, everything else at 0)"""
  z = np.zeros(np.shape(p))
  return {"sgd": (None, None), "momentum": (z, None), "momentum_cosine": (z, None), "rmsprop": (z + 1.0, z),
          "adam": (z, z)}[kind]


def _hyper(spec):
  """(kind, hyperparameters as the fp32 values an update uses), defaults taken from the oracle's optimizers"""
  o = orc.make_optimizer(spec)
  kind = spec[0]
  h = {"sgd": lambda: [o.lr], "momentum": lambda: [o.lr, o.m], "momentum_cosine": lambda: [o.lr0, o.m, o.decay_steps, o.alpha],
       "rmsprop": lambda: [o.lr, o.rho, o.mu, o.eps], "adam": lambda: [o.lr, o.b1, o.b2, o.eps]}[kind]()
  return kind, [float(np.float32(v)) for v in h]


def opt_update(spec, p, g, s0, s1, step):
  """TF1 rule in float64 -> (p', s0', s1', bounds of each); hyperparameters as the fp32 values the kernel receives"""
  kind, h = _hyper(spec)
  p, g = f64(p), f64(g)
  s0 = None if s0 is None else f64(s0)
  s1 = None if s1 is None else f64(s1)
  out = dict(s0=None, s1=None, s0_b=None, s1_b=None)
  if kind == "sgd":
    d = h[0] * g
    out.update(p=p - d, p_b=2 * U * (np.abs(p) + 2 * np.abs(d)))
  elif kind in ("momentum", "momentum_cosine"):
    a = h[1] * s0 + g
    a_b = 2 * U * (np.abs(h[1] * s0) + np.abs(g) + np.abs(a))
    lr, lr_b = h[0], 2 * U * h[0]
    if kind == "momentum_cosine":
      dsteps, alpha = h[2], h[3]
      st = min(float(step), dsteps)
      cos = 0.5 * (1 + math.cos(math.pi * st / dsteps))
      lr = h[0] * ((1 - alpha) * cos + alpha)
      lr_b = h[0] * (1 - alpha) * 8 * U + 4 * U * lr
    d = lr * a
    out.update(p=p - d, p_b=2 * U * (np.abs(p) + 2 * np.abs(d)) + lr * a_b + lr_b * np.abs(a), s0=a, s0_b=a_b)
  elif kind == "rmsprop":
    lr, rho, mu, eps = h
    ms = rho * s0 + (1 - rho) * g * g
    ms_b = 3 * U * (np.abs(rho * s0) + (1 - rho) * g * g)
    q = lr * g / np.sqrt(ms + eps)
    mom = mu * s1 + q
    mom_b = 3 * U * (np.abs(mu * s1) + 2 * np.abs(q)) + np.abs(q) * ms_b / (2 * (ms + eps))
    out.update(p=p - mom, p_b=2 * U * (np.abs(p) + np.abs(mom)) + mom_b, s0=ms, s0_b=ms_b, s1=mom, s1_b=mom_b)
  else:
    lr, b1, b2, eps = h
    t = float(step + 1)
    b1t, b2t = b1 ** t, b2 ** t
    lr_t = lr * math.sqrt(1 - b2t) / (1 - b1t)
    # powf is within ~2 ulp of b^t; 1 - b^t magnifies that by b^t / (1 - b^t)
    lr_t_b = lr_t * (8 * U + 4 * U * b2t / (1 - b2t) + 4 * U * b1t / (1 - b1t))
    m = s0 + (1 - b1) * (g - s0)
    m_b = 3 * U * (np.abs(s0) + (1 - b1) * (np.abs(g) + np.abs(s0)))
    v = s1 + (1 - b2) * (g * g - s1)
    v_b = 3 * U * (np.abs(s1) + (1 - b2) * (g * g + np.abs(s1)))
    den = np.sqrt(v) + eps
    d = lr_t * m / den
    sq_b = np.where(v > 0, v_b / (2 * np.sqrt(np.maximum(v, 1e-300))), np.sqrt(v_b)) + U * np.sqrt(v)
    d_b = (lr_t_b * np.abs(m) + lr_t * m_b) / den + np.abs(d) * (sq_b / den + 4 * U)
    out.update(p=p - d, p_b=2 * U * (np.abs(p) + np.abs(d)) + d_b, s0=m, s0_b=m_b, s1=v, s1_b=v_b)
  return out


def ema_update(state, x, decay):
  """zero-debiased EMA (candidate.py:117-129) of the adanet loss x -> (state', bound)"""
  d = float(np.float32(decay))
  b, n = float(state[0]), float(state[1])
  b2 = b - (b - x) * (1 - d)
  n2 = n + 1
  f = 1 - d ** n2
  v = b2 / f
  b_b = 3 * U * (abs(b) + abs(x))
  v_b = abs(v) * (4 * U + 4 * U * d ** n2 / f) + b_b / f
  return np.array([b2, n2, v]), np.array([b_b, 0.0, v_b])


# ------------------------------------------------------------------------------------------------------------------
# CPU: the float64 step against the fp32 oracle (no GPU)
# ------------------------------------------------------------------------------------------------------------------
class _StepList(list):
  """a trace list whose length is the dropout step orc.train_step draws the mask for"""

  def __init__(self, n):
    super().__init__()
    self.n = n

  def __len__(self):
    return self.n


def _gammas(ens, cxs):
  lam, beta = float(ens.get("adanet_lambda", 0.0)), float(ens.get("adanet_beta", 0.0))
  if lam == 0.0 and beta == 0.0:
    return [0.0] * len(cxs)
  return [float(orc.adanet_gamma(c, lam, beta)) for c in cxs]


def _rand_state(cands, rng, opt_step):
  """the pre-step optimizer / EMA state the CPU check starts from: nonzero slots, counters far from 0"""
  out = []
  for c in cands:
    params = [a for w, b in zip(*c["p"]) for a in (w, b)]
    kind = c["opt"][0]
    s0 = s1 = None
    if kind in ("momentum", "momentum_cosine"):
      s0 = [(rng.standard_normal(p.shape) * 0.01).astype(np.float32) for p in params]
    elif kind == "rmsprop":
      s0 = [rng.uniform(0.05, 2.0, p.shape).astype(np.float32) for p in params]
      s1 = [(rng.standard_normal(p.shape) * 0.01).astype(np.float32) for p in params]
    elif kind == "adam":
      s0 = [(rng.standard_normal(p.shape) * 0.01).astype(np.float32) for p in params]
      s1 = [(rng.uniform(0, 1e-2, p.shape) ** 2).astype(np.float32) for p in params]
    out.append(dict(s0=s0, s1=s1, step=opt_step))
  return out


def _oracle_opt(spec, st):
  o = orc.make_optimizer(spec)
  kind = spec[0]
  if kind in ("momentum", "momentum_cosine"):
    o.acc = [a.copy() for a in st["s0"]]
  if kind == "momentum_cosine":
    o.t = st["step"]
  if kind == "rmsprop":
    o.ms, o.mom = [a.copy() for a in st["s0"]], [a.copy() for a in st["s1"]]
  if kind == "adam":
    o.m, o.v, o.t = [a.copy() for a in st["s0"]], [a.copy() for a in st["s1"]], st["step"]
  return o


def reference_step(case, frozen, cands, mix, bias, opt_states, ema_state, x, y, step_dev, floor=0.0, relu_masks=None):
  """One whole step in float64 from an explicit state: returns per candidate the forward, head, gradients and next
  parameters / slots / EMA.  relu_masks[k]: the backward masks of candidate k's hidden layers, taken from another
  implementation's forward so that a pre-activation within rounding of 0 cannot put the two on opposite sides of the
  ReLU's kink."""
  ens = case["ens"]
  mt = ens.get("mixture_weight_type", "scalar")
  f_logits = []
  for f in frozen:
    h = f64(x)
    for i, (w, b) in enumerate(zip(*f["p"])):
      h, _ = layer_fwd(h, w, b, i < len(f["p"][0]) - 1)
    f_logits.append(h)
  res = []
  for k, c in enumerate(cands):
    ws, bs = c["p"]
    hs, masks, muls = [f64(x)], [None], [1.0]
    for i, (w, b) in enumerate(zip(ws, bs)):
      last = i == len(ws) - 1
      d = c.get("dropout")[i] if (c.get("dropout") and not last and i < len(c["dropout"])) else None
      keep = orc.dropout_keep_mask(d[1], i, step_dev, x.shape[0], w.shape[1], d[0]) if d else None
      h, _ = layer_fwd(hs[-1], w, b, not last, keep, d[0] if d else 0.0)
      hs.append(h)
      if not last:
        masks.append(h > 0)
        muls.append(1.0 / (1.0 - float(np.float32(d[0]))) if d else 1.0)
    logits = hs[-1]
    if relu_masks is not None:
      masks = [None] + list(relu_masks[k])
    loss, _, dl, _ = head_loss(case["head"], logits, y)
    gam = _gammas(ens, [f["cx"] for f in frozen] + [c["cx"]])
    eh = ensemble(case["head"], mt, mix[k], bias[k], f_logits + [logits], y, gam,
                  1.0 if ens.get("legacy_train_op") else 2.0, ens.get("use_bias", False))
    bw = backward(ws, hs[:-1], dl, masks, muls)
    bw["db"][len(ws) - 1] = dl.sum(axis=0)
    grads = [a for dw, db in zip(bw["dw"], bw["db"]) for a in (dw, db)]
    params = [a for w, b in zip(ws, bs) for a in (w, b)]
    st = opt_states[k]
    ups = [opt_update(c["opt"], p, g, st["s0"][j] if st["s0"] else None, st["s1"][j] if st["s1"] else None, st["step"])
           for j, (p, g) in enumerate(zip(params, grads))]
    ens_up = None
    if ens.get("optimizer") is not None:
      eg = [eh["dmw"]] + ([eh["db"]] if ens.get("use_bias") else [])
      ep = [mix[k]] + ([bias[k]] if ens.get("use_bias") else [])
      ens_up = [opt_update(ens["optimizer"], p, g, *_fresh_slots(ens["optimizer"][0], p), 0) for p, g in zip(ep, eg)]
    ema, _ = ema_update(ema_state[k], eh["out3"][2], 0.9)
    res.append(dict(hs=hs, loss=loss, dl=dl, eh=eh, bw=bw, ups=ups, ens_up=ens_up, ema=ema))
  return res


CPU_B = {"b4097": 129, "b4096_w1024": 64}      # the large-batch cases at a batch the CPU check can afford


@pytest.mark.parametrize("name", ["mixed", "vector_warm", "vector_warm_legacy", "mse", "sigmoid", "dropout", "b37", "b4097",
                                  "b4096_w1024", "opt_state"])
def test_reference_step_matches_oracle(name):
  """The float64 step and orc.train_step (fp32) agree from the same state, to fp32 level, on every tensor the GPU test
  checks: the restatement means what the oracle means.  The state has nonzero optimizer slots, counters far from 0
  (Adam at 10^5; Momentum-cosine before, at and after decay_steps) and, for the dropout case, a step past 2^32."""
  case = dict(CASES[name], B=CPU_B.get(name, CASES[name]["B"]))
  frozen, cands, warm = _case_data(case, seed=5)
  ens = case["ens"]
  mt = ens.get("mixture_weight_type", "scalar")
  C, B = case["C"], case["B"]
  rng = np.random.default_rng(9)
  step = 2 ** 32 + 3 if name == "dropout" else 7
  opt_states = _rand_state(cands, rng, DECAY + 3)
  for k, c in enumerate(cands):
    if c["opt"][0] == "adam":
      opt_states[k]["step"] = 10 ** 5
    if c["opt"][0] == "momentum_cosine":
      opt_states[k]["step"] = DECAY + (-1, 0, 5)[k % 3]
  nm = len(frozen) + 1
  mix, bias = [], []
  for _ in cands:
    m = np.full((nm,) if mt == "scalar" else (nm, C), 1.0 / nm, dtype=np.float32)
    bv = np.zeros((C,), np.float32)
    if warm is not None:
      m[:len(frozen)] = warm[0]
      bv = warm[1].copy()
    mix.append(m)
    bias.append(bv)
  ema0 = [np.array([2.1, 4.0, 2.0], dtype=np.float32) for _ in cands]
  x, y = _batch(case, 0)
  o_masks = [[a > 0 for a in orc.mlp_forward(c["p"][0], c["p"][1], x, (c["dropout"], step) if c.get("dropout") else None)[1:-1]]
             for c in cands]
  ref = reference_step(case, frozen, cands, mix, bias, opt_states, ema0, x, y, step, relu_masks=o_masks)
  # the oracle from the same state
  o_frozen = [orc.FrozenMember(0, "f%d" % k, f["p"][0], f["p"][1], f["cx"]) for k, f in enumerate(frozen)]
  o_ens = orc.EnsemblerSpec(**ens)
  o_cands = []
  for k, c in enumerate(cands):
    spec = orc.SubnetworkSpec(c["name"], c["dims"], c["cx"], c["opt"], ws=c["p"][0], bs=c["p"][1], dropout=c.get("dropout"))
    ema = orc.ZeroDebiasEMA(0.9)
    ema.biased, ema.n, ema.value = np.float32(ema0[k][0]), int(ema0[k][1]), np.float32(ema0[k][2])
    cs = orc.CandidateState("c%d" % k, spec, [w.copy() for w in c["p"][0]], [b.copy() for b in c["p"][1]],
                            _oracle_opt(c["opt"], opt_states[k]),
                            [np.array(mix[k][j], dtype=np.float32) for j in range(nm)], bias[k].copy(),
                            orc.make_optimizer(ens.get("optimizer")), ema, [f["cx"] for f in frozen] + [c["cx"]])
    cs.trace_sub_loss = _StepList(step)
    o_cands.append(cs)
  orc.train_step(o_cands, o_frozen, o_ens, x, y, case["head"])

  def close(got, want, what):
    got, want = f64(got), f64(want)
    err = np.abs(got - want).max() if got.size else 0.0
    assert err <= 2e-5 * max(np.abs(want).max(), 1e-3), "%s %s: max err %.3g against %.3g" % (name, what, err, np.abs(want).max())

  for k, (r, o) in enumerate(zip(ref, o_cands)):
    close(o.trace_sub_loss[-1], r["loss"], "cand %d sub_loss" % k)
    close(o.trace_ens_loss[-1], r["eh"]["out3"][0], "cand %d ens_loss" % k)
    close(o.trace_adanet_loss[-1], r["eh"]["out3"][2], "cand %d adanet_loss" % k)
    close(o.trace_ema[-1], r["ema"][2], "cand %d ema" % k)
    for j, (w, b) in enumerate(zip(o.ws, o.bs)):
      close(w, r["ups"][2 * j]["p"], "cand %d w%d" % (k, j))
      close(b, r["ups"][2 * j + 1]["p"], "cand %d b%d" % (k, j))
    so = o.sub_opt
    slots = {"momentum": [("acc", "s0")], "momentum_cosine": [("acc", "s0")], "rmsprop": [("ms", "s0"), ("mom", "s1")],
             "adam": [("m", "s0"), ("v", "s1")]}.get(cands[k]["opt"][0], [])
    for attr, key in slots:
      for j, a in enumerate(getattr(so, attr)):
        close(a, r["ups"][j][key], "cand %d %s %d" % (k, attr, j))
    if r["ens_up"] is not None:
      for j in range(nm):
        close(o.weights[j], r["ens_up"][0]["p"][j], "cand %d mixture weight %d" % (k, j))
      if ens.get("use_bias"):
        close(o.bias, r["ens_up"][1]["p"], "cand %d ensemble bias" % k)


def test_oracle_bagged_prepass_draws_dropout():
  """A bagged subnetwork's own train op runs in TRAIN mode (its secondary session.run, autoensemble/common.py:43-56),
  so orc.train_step's pre-pass draws the step's dropout mask, as the engine's pre-pass does: the weights after the
  step equal a float64 SGD step on the own minibatch through the masked forward, and not the unmasked one."""
  case = CASES["bagging"]
  frozen, cands, _ = _case_data(case, seed=5)
  c = cands[0]
  ws, bs = c["p"]
  x, y = _batch(case, 0)
  xo, yo = _batch(case, 500)
  step = 9
  lr = float(np.float32(c["opt"][1]))

  def sgd_step(dropout):
    hs, masks, muls = [f64(xo)], [None], [1.0]
    for i, (w, b) in enumerate(zip(ws, bs)):
      d = _drop(dict(dropout=dropout), i, len(ws))
      keep = orc.dropout_keep_mask(d[1], i, step, xo.shape[0], w.shape[1], d[0]) if d else None
      h, _ = layer_fwd(hs[-1], w, b, i < len(ws) - 1, keep, d[0] if d else 0.0)
      hs.append(h)
      if i < len(ws) - 1:
        masks.append(h > 0)
        muls.append(_dx_mul(d))
    _, _, g, _ = head_loss(case["head"], hs[-1], yo)
    bw = backward(ws, hs[:-1], g, masks, muls)
    bw["db"][-1] = g.sum(axis=0)
    return [f64(w) - lr * dw for w, dw in zip(ws, bw["dw"])], [f64(b) - lr * db for b, db in zip(bs, bw["db"])]

  want_w, want_b = sgd_step(c["dropout"])
  plain_w, _ = sgd_step(None)
  o_frozen = [orc.FrozenMember(0, "f%d" % k, f["p"][0], f["p"][1], f["cx"]) for k, f in enumerate(frozen)]
  spec = orc.SubnetworkSpec(c["name"], c["dims"], c["cx"], c["opt"], ws=ws, bs=bs, dropout=c["dropout"])
  o_ens = orc.EnsemblerSpec(**case["ens"])
  cs = orc.build_candidates(0, [spec], o_frozen, o_ens, case["C"], 0.9)[0]
  cs.trace_sub_loss = _StepList(step)
  orc.train_step([cs], o_frozen, o_ens, x, y, case["head"], own_batches={0: (xo, yo)})
  for i, (w, b) in enumerate(zip(cs.ws, cs.bs)):
    assert np.abs(f64(w) - want_w[i]).max() <= 2e-5 * np.abs(want_w[i]).max(), "w%d" % i
    assert np.abs(f64(b) - want_b[i]).max() <= 2e-5 * max(np.abs(want_b[i]).max(), 1e-3), "b%d" % i
  assert np.abs(want_w[0] - plain_w[0]).max() > 100 * 2e-5 * np.abs(want_w[0]).max()     # the mask matters here


# ------------------------------------------------------------------------------------------------------------------
# GPU: teacher-forced steps of the engine
# ------------------------------------------------------------------------------------------------------------------
REPORT = {}
_FMT = ["f16"]              # the plane format of the module parameter running


def _note(stage, got, exact, bound):
  err = np.abs(f64(got) - exact)
  r = float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), np.where(err > 0, np.inf, 0.0)))) if err.size else 0.0
  _report(stage, r)


def _report(stage, value):
  key = (_FMT[0], stage)
  REPORT[key] = max(REPORT.get(key, 0.0), value)


def _check(fails, stage, got, exact, bound, what):
  got = np.asarray(got)
  exact, bound = np.broadcast_to(f64(exact), got.shape), np.broadcast_to(f64(bound), got.shape)
  _note(stage, got, exact, bound)
  fails += _cw(got, exact, bound, what)


@pytest.fixture(scope="module", params=["f16", "tf32"])
def fmt(request):
  import torch
  from tests.test_gpu_plane_groups import _open, _set_format
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _set_format(_lib, request.param)
  _lib.plane_overflow()
  _FMT[0] = request.param
  yield request.param
  _lib.set_plane_format(before)


@pytest.fixture(scope="module", autouse=True)
def _print_report():
  yield
  for f in sorted({f for f, _ in REPORT}):
    print("\n%s planes: " % f + ", ".join("%s %.3g" % (st, v) for (ff, st), v in sorted(REPORT.items()) if ff == f))


def _merge(net_planes, rows, cols):
  import torch
  from adanet_b200 import _lib
  out = torch.empty((rows, cols), dtype=torch.float32, device="cuda")
  _lib.check(_lib.load().adn_planes_merge(net_planes.data_ptr(), rows, cols, out.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream), "adn_planes_merge")
  return out.cpu().numpy()


def _plane_checks(fails, t, rows, cols, got, what):
  """sign bits = the stored values > 0, and zero K padding"""
  from tests.test_gpu_planes import _layout
  from tests.test_gpu_plane_groups import _bits_of
  from adanet_b200 import _lib
  hi, bits, bk = _layout(_lib, t, rows, cols)
  if cols % bk and not (hi[-1, :, cols % bk:] == 0).all():
    fails.append("%s: K padding of the planes is not zero" % what)
  pos = np.zeros((rows, bits.shape[0] * 32), dtype=bool)
  pos[:, :cols] = got > 0
  if not np.array_equal(bits, _bits_of(pos)):
    fails.append("%s: sign bits disagree with the stored values" % what)


def _build_plan(case, frozen, cands, warm, trace_capacity=4096, shards=None, batch=None):
  import torch
  from adanet_b200.core import engine as eng
  dev = torch.device("cuda", torch.cuda.current_device())
  B = batch or case["B"]
  fnets = [eng.DenseNet("frozen%d" % k, f["dims"], f["p"][0], f["p"][1], f["cx"], B, dev, iteration=0)
           for k, f in enumerate(frozen)]
  specs = [eng.SubnetworkPlanSpec(c["name"], c["dims"], c["cx"], c["opt"], [w.copy() for w in c["p"][0]],
                                  [b.copy() for b in c["p"][1]], dropout=c.get("dropout"), image_shape=c.get("image"),
                                  own_input=c.get("own", False)) for c in cands]
  ens = eng.EnsemblerPlanSpec(**case["ens"])
  ec = None
  if case.get("heads"):
    others = {k: eng.EnsemblerPlanSpec(**v) for k, v in case["ensemblers"].items()}
    ec = [(g, name, b, keep, others[e] if e else None) for g, (name, b, keep, e) in enumerate(case["heads"])]
  plan = eng.IterationPlan(1 if frozen else 0, specs, fnets, ens, B, case.get("input", D), case["C"], case["head"],
                           trace_capacity=trace_capacity, device=dev,
                           prev_mixture_weights=warm[0] if warm else None, prev_bias=warm[1] if warm else None,
                           shards=shards, ensemble_candidates=ec)
  return plan, fnets


def _frozen_snapshot(fnets):
  return [[t.clone() for t in f.ws + f.bs + (f.wps or [])] for f in fnets]


def _acts(net, B, planes):
  """a net's hidden activations as dense fp32: merged from their planes, or the SIMT path's dense buffers"""
  return [(_merge(net.hp[i], B, d) if planes else net.acts[i].cpu().numpy()) for i, d in enumerate(net.dims[1:-1])]


def _engine_fwd(c, B, x):
  """the engine's hidden activations (merged from their planes) and logits; hs[0] = x"""
  return [f64(x)] + _acts(c.net, B, True), c.net.logits.cpu().numpy()


def _drop(spec, i, n):
  """(rate, seed) of hidden layer i of a candidate spec, or None"""
  return spec["dropout"][i] if (spec.get("dropout") and i < n - 1 and i < len(spec["dropout"])) else None


def _dx_mul(d):
  """the factor on the gradient below a dropped-out layer: 1 / (1 - rate), from the spec's rate"""
  return 1.0 / (1.0 - float(np.float32(d[0]))) if d else 1.0


def check_forward(fails, case, c, spec, wsrc, x_in, step_dev, floor, tag, planes=True):
  """every layer of candidate c from the engine's own input to it, with the weights in `wsrc` (the state before the
  step, or after it for a bagged subnetwork's main pass); returns (hs, masks, dx_muls, logits)"""
  B = c.batch
  hs = [f64(x_in)] + _acts(c.net, B, planes)
  logits = c.net.logits.cpu().numpy()
  n = len(c.net.ws)
  masks, muls = [None], [1.0]
  for i in range(n):
    w, b = wsrc["c%d_w%d" % (c.index, i)], wsrc["c%d_b%d" % (c.index, i)]
    last = i == n - 1
    d = _drop(spec, i, n)
    keep = orc.dropout_keep_mask(d[1], i, step_dev, B, w.shape[1], d[0]) if d else None
    exact, bound = layer_fwd(hs[i], w, b, not last, keep, float(np.float32(d[0])) if d else 0.0, floor, fp32_dot=not planes)
    what = "%s layer %d (%d -> %d%s)" % (tag, i, w.shape[0], w.shape[1], ", dropout" if d else "")
    got = logits if last else hs[i + 1]
    _check(fails, "forward", got, exact, bound, what)
    if not last:
      if planes:
        _plane_checks(fails, c.net.hp[i], B, w.shape[1], got, what)
      if d is not None:
        pre_drop, pb = layer_fwd(hs[i], w, b, True, None, 0.0, floor)
        if not (got[~keep] == 0).all():
          fails.append("%s: a dropped entry is nonzero" % what)
        clear = pre_drop > 2 * pb
        if not np.array_equal(got[clear] != 0, keep[clear]):
          fails.append("%s: the dropout mask differs from orc.dropout_keep_mask" % what)
      masks.append(got > 0)
      muls.append(_dx_mul(d))
  return hs, masks, muls, logits


def check_frozen_forward(fails, fnets, frozen, x, floor, planes=True):
  for k, (f, fs) in enumerate(zip(fnets, frozen)):
    h = f64(x)
    ws, bs = fs["p"]
    if f.stem:
      # a frozen SimpleCNN member: its conv stem from the minibatch, its dense layers from the engine's pooled features
      st = conv_stem64(np.asarray(x).reshape((f.batch,) + tuple(f.image_shape)), ws[0], bs[0])
      h = _merge(f.stem_out, f.batch, f.dims[0])
      _check(fails, "forward", h, st["pooled"], st["bound"] + floor, "frozen %d conv stem" % k)
      ws, bs = ws[1:], bs[1:]
    acts = _acts(f, f.batch, planes)
    for i, (w, b) in enumerate(zip(ws, bs)):
      last = i == len(ws) - 1
      exact, bound = layer_fwd(h, w, b, not last, floor=floor, fp32_dot=not planes)
      got = f.logits.cpu().numpy() if last else acts[i]
      _check(fails, "forward", got, exact, bound, "frozen %d layer %d" % (k, i))
      h = got


def check_heads(fails, case, c, logits, y, tag, fp32_dot=False):
  """sub_out3[0], dlogits and the logits layer's db from the engine's logits; returns the engine's dlogits"""
  loss, lb, g, gb = head_loss(case["head"], logits, y)
  _check(fails, "heads", c.sub_out3[:1].cpu().numpy(), loss, lb, tag + " sub_loss")
  dl = c.dlogits.cpu().numpy()
  _check(fails, "heads", dl, g, gb, tag + " dlogits")
  dlf = f64(dl)
  _check(fails, "heads", c.dbs[-1].cpu().numpy(), dlf.sum(axis=0), _tol(c.batch, fp32_dot) * np.abs(dlf).sum(axis=0),
         tag + " logits-layer db")
  return dl


def check_backward(fails, c, pre, hs, masks, muls, dl, floor_g, floor_x, tag, deep=False, fp32_dot=False, dx0=False):
  n = len(c.net.ws)
  ws = [pre["c%d_w%d" % (c.index, i)] for i in range(n)]
  bw = backward(ws, hs, dl, masks, muls, floor_g, floor_x, fp32_dot=fp32_dot, dx0=dx0)
  if deep and floor_g:
    # what the fp16 floor costs a deep net: per layer, the median over dW entries of (floor's bound) / |dW| -- the
    # relative accuracy left to that entry by the floor alone -- and the largest share of a bound that is floor
    fb = backward(ws, hs, dl, masks, muls, floor_g, floor_x, tol=0.0)["dw_b"]
    rel = [float(np.median(f[np.abs(d) > 0] / np.abs(d[np.abs(d) > 0]))) for f, d in zip(fb, bw["dw"])]
    share = [float(np.max(f[b > 0] / b[b > 0])) for f, b in zip(fb, bw["dw_b"])]
    _report("deep dW: median floor/|dW| in the worst layer", max(rel))
    _report("deep dW: largest floor share of a bound", max(share))
  for i in range(n):
    _check(fails, "backward", c.dws[i].cpu().numpy(), bw["dw"][i], bw["dw_b"][i], "%s dW%d" % (tag, i))
    if i < n - 1:
      _check(fails, "backward", c.dbs[i].cpu().numpy(), bw["db"][i], bw["db_b"][i], "%s db%d" % (tag, i))
  return bw


def _slots(pre, prefix, j):
  s0 = pre.get("%ss0_%d" % (prefix, j))
  s1 = pre.get("%ss1_%d" % (prefix, j))
  return s0, s1


def check_update(fails, opt_spec, params_pre, grads, pre, post, prefix, names, tag, slot_index=None, grad_err=None):
  """TF1 rule on the engine's gradients; slots; exact step counter.  slot_index[j]: the optimizer's tensor index of
  names[j] (default j); grad_err[j]: a bound on the error of grads[j] when it is not the engine's own buffer."""
  step = int(pre[prefix + "step"]) if (prefix + "step") in pre else 0
  for j, (p, g, nm) in enumerate(zip(params_pre, grads, names)):
    t = slot_index[j] if slot_index is not None else j
    s0, s1 = _slots(pre, prefix, t)
    up = opt_update(opt_spec, p, g, s0, s1, step)
    got = post[nm]
    pb = up["p_b"]
    if grad_err is not None and grad_err[j] is not None:
      assert opt_spec[0] == "sgd"
      pb = pb + _hyper(opt_spec)[1][0] * grad_err[j]
    _check(fails, "update", got, up["p"].reshape(got.shape), pb.reshape(got.shape), "%s %s" % (tag, nm))
    for key in ("s0", "s1"):
      if up[key] is not None:
        gk = post["%s%s_%d" % (prefix, key, t)]
        _check(fails, "update", gk, up[key].reshape(gk.shape), up[key + "_b"].reshape(gk.shape), "%s %s slot %s" % (tag, nm, key))
  if (prefix + "step") in pre and int(post[prefix + "step"]) != step + 1:
    fails.append("%s: optimizer step %d -> %d" % (tag, step, int(post[prefix + "step"])))


def _planes_words(rows, cols):
  """32-bit words of the hi and lo planes of a [rows, cols] plane tensor (the sign-bit words follow them)"""
  from adanet_b200 import _lib
  f16 = _lib.plane_format() == _lib.PLANES_F16
  bk = 64 if f16 else 32
  elems = -(-(-(-cols // bk) * rows * bk) // 128) * 128
  return elems if f16 else 2 * elems


def check_planes_resplit(fails, pairs, tag):
  """The hi / lo planes the optimizer wrote = a fresh split of the updated weights, byte for byte.  (The optimizer
  leaves a weight tensor's sign-bit words alone: a weight is only ever the B operand of a GEMM, and the ReLU masks
  come from the activations' sign bits.)  pairs: [(name, weights, their planes)]"""
  import torch
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  lib = _lib.load()
  for name, w, wp in pairs:
    fresh = eng.new_planes(w.shape[0], w.shape[1], w.device)
    _lib.check(lib.adn_planes_split(w.data_ptr(), w.shape[0], w.shape[1], fresh.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream), "adn_planes_split")
    n = _planes_words(w.shape[0], w.shape[1])
    if not torch.equal(fresh[:n].view(torch.int32), wp[:n].view(torch.int32)):
      fails.append("%s: the planes of %s the optimizer wrote differ from its split" % (tag, name))


def check_bookkeeping(fails, h, pre, post, key, step_dev, sub_loss, cap, tag):
  ema_pre = pre[key + "ema_state"]
  out3 = h.out3.cpu().numpy()
  want, wb = ema_update(ema_pre, float(out3[2]), h.decay)
  _check(fails, "update", post[key + "ema_state"], want, wb, tag + " ema_state")
  row = post[key + "trace"][step_dev % cap]
  exp = np.array([sub_loss, out3[0], out3[2], post[key + "ema_state"][2]], dtype=np.float32)
  if not np.array_equal(row, exp, equal_nan=True):
    fails.append("%s: trace row %d is %s, want %s" % (tag, step_dev % cap, row, exp))


def conv_stem64(images, k, b):
  """float64 conv3x3 "same" + bias + ReLU + maxpool 2x2 + flatten (orc.conv_stem_forward's arithmetic) with its
  componentwise bound, the im2col patches, the pool arg-max and the windows whose arg-max is within rounding of a tie"""
  x = f64(images)
  n, h, w, cin = x.shape
  f = k.shape[3]
  pad = np.zeros((n, h + 2, w + 2, cin))
  pad[:, 1:-1, 1:-1, :] = x
  patches = np.stack([pad[:, ky:ky + h, kx:kx + w, :] for ky in range(3) for kx in range(3)], axis=3).reshape(n * h * w, 9 * cin)
  kk = f64(k).reshape(9 * cin, f)
  conv = patches @ kk + f64(b)
  cb = TOL * (np.abs(patches) @ np.abs(kk) + np.abs(f64(b)))
  win = lambda t: t.reshape(n, h // 2, 2, w // 2, 2, f).transpose(0, 1, 3, 2, 4, 5).reshape(n, h // 2, w // 2, 4, f)
  cw, bw = win(conv), win(cb)
  arg = cw.argmax(axis=3)
  top = np.sort(cw, axis=3)
  amb = (top[:, :, :, -1] - top[:, :, :, -2]) <= 2 * bw.max(axis=3)
  pooled = np.maximum(cw.max(axis=3), 0.0)
  return dict(pooled=pooled.reshape(n, -1), bound=bw.max(axis=3).reshape(n, -1), patches=patches, arg=arg, amb=amb,
              shape=(n, h, w, cin, f))


def check_stem_grads(fails, st, dpool, dk, db, tag):
  """kernel / bias gradients from the engine's pooled-feature gradient: each gradient routed to its window's arg-max;
  a window within rounding of a tie may route to any of its four positions, which the bound allows for"""
  n, h, w, cin, f = st["shape"]
  g = f64(dpool).reshape(n, h // 2, w // 2, f)
  dwin = np.zeros((n, h // 2, w // 2, 4, f))
  np.put_along_axis(dwin, st["arg"][:, :, :, None, :], g[:, :, :, None, :], axis=3)
  awin = np.repeat((np.abs(g) * st["amb"])[:, :, :, None, :], 4, axis=3)
  unwin = lambda t: t.reshape(n, h // 2, w // 2, 2, 2, f).transpose(0, 1, 3, 2, 4, 5).reshape(n * h * w, f)
  dconv, aconv = unwin(dwin), unwin(awin)
  P = np.abs(st["patches"])
  exact = (st["patches"].T @ dconv).reshape(3, 3, cin, f)
  bound = (TOL * (P.T @ np.abs(dconv)) + 2 * P.T @ aconv).reshape(3, 3, cin, f)
  _check(fails, "backward", dk, exact, bound, tag + " conv stem dK")
  _check(fails, "backward", db, dconv.sum(axis=0), TOL * np.abs(dconv).sum(axis=0) + 2 * aconv.sum(axis=0), tag + " conv stem db")


def check_candidate(fails, case, c, spec, pre, post, x, y, step_dev, tag, planes, f16):
  """forward, the subnetwork's own head, backward (+ the conv stem's) and the update of one trained candidate"""
  key = "c%d_" % c.index
  B, n = c.batch, len(c.net.ws)
  floor_x = F16_FLOOR if f16 else 0.0
  floor_g = F16_FLOOR * 2.0 ** -c.dz_log2 if f16 else 0.0
  x_in, st = x, None
  if c.net.stem:
    st = conv_stem64(x.reshape((B,) + tuple(spec["image"])), pre[key + "stem_k"], pre[key + "stem_b"])
    x_in = _merge(c.net.stem_out, B, c.net.dims[0])
    _check(fails, "forward", x_in, st["pooled"], st["bound"] + floor_x, tag + " conv stem")
    _plane_checks(fails, c.net.stem_out, B, c.net.dims[0], x_in, tag + " conv stem")
  hs, masks, muls, logits = check_forward(fails, case, c, spec, pre, x_in, step_dev, floor_x, tag, planes)
  dl = check_heads(fails, case, c, logits, y, tag, not planes)
  if st is not None:
    masks[0] = f64(x_in) > 0             # the pooled features' sign bits: ReLU and the pool's routing
  bw = check_backward(fails, c, pre, hs, masks, muls, dl, floor_g, floor_x, tag, deep=spec.get("deep", False),
                      fp32_dot=not planes, dx0=st is not None)
  names = [key + nm for i in range(n) for nm in ("w%d" % i, "b%d" % i)]
  grads = [t.cpu().numpy() for i in range(n) for t in (c.dws[i], c.dbs[i])]
  if st is not None:
    dpool = c.dpool.cpu().numpy()
    _check(fails, "backward", dpool, bw["dx"], bw["dx_b"], tag + " dpool (the first dense layer's dX)")
    dk, db = c.d_stem_k.cpu().numpy(), c.d_stem_b.cpu().numpy()
    check_stem_grads(fails, st, dpool, dk, db, tag)
    names = [key + "stem_k", key + "stem_b"] + names
    grads = [dk, db] + grads
  check_update(fails, spec["opt"], [pre[nm] for nm in names], grads, pre, post, key + "sub_opt_", names, tag)
  if planes:
    check_planes_resplit(fails, [("W%d" % i, w, wp) for i, (w, wp) in enumerate(zip(c.net.ws, c.net.wps))], tag)


def check_bagged(fails, case, c, spec, pre, post, own, x, y, step_dev, tag, f16):
  """A bagged subnetwork: its step on its own minibatch runs before the main pass (pre-pass, dropout drawn for the
  same step), whose activations the main pass then overwrites.  So the pre-pass forward is float64 from the state
  before the step, with its error bound carried layer by layer and every mask entry within rounding of 0 treated as
  either way; its gradient buffers (but the logits layer's db, which the main pass's head rewrites) and the update
  follow from it.  The main pass's forward must use the UPDATED weights, and its head is checked as usual."""
  key = "c%d_" % c.index
  xo, yo = own
  n = len(c.net.ws)
  floor_x = F16_FLOOR if f16 else 0.0
  floor_g = F16_FLOOR * 2.0 ** -c.dz_log2 if f16 else 0.0
  h, E = f64(xo), np.zeros(xo.shape)
  hs, errs, masks, ambs, muls = [h], [None], [None], [None], [1.0]
  ws = [pre[key + "w%d" % i] for i in range(n)]
  for i in range(n):
    w, b = f64(ws[i]), f64(pre[key + "b%d" % i])
    z = h @ w + b
    zb = TOL * (np.abs(h) @ np.abs(w) + np.abs(b)) + E @ np.abs(w)
    if floor_x:
      zb += floor_x * (np.abs(w).sum(axis=0)[None, :] + np.abs(h).sum(axis=1)[:, None] + 1.0)
    if i == n - 1:
      logits, lerr = z, zb
      break
    d = _drop(spec, i, n)
    keep = orc.dropout_keep_mask(d[1], i, step_dev, xo.shape[0], w.shape[1], d[0]) if d else np.ones(z.shape, bool)
    s = _dx_mul(d)
    h = np.where(keep, np.maximum(z, 0.0) * s, 0.0)
    E = np.where(keep, zb * s, 0.0)
    hs.append(h)
    errs.append(E)
    masks.append(h > 0)
    ambs.append(((np.abs(z) <= zb) & keep).astype(np.float64))
    muls.append(s)
  loss, lb, g, gb = head_loss(case["head"], logits, yo, lerr)
  _check(fails, "heads", c.own_loss.cpu().numpy(), loss, lb, tag + " pre-pass loss")
  bw = backward(ws, hs, g, masks, muls, floor_g, floor_x, h_err=errs, amb=ambs, dz_err=gb)
  for i in range(n):
    _check(fails, "backward", c.dws[i].cpu().numpy(), bw["dw"][i], bw["dw_b"][i], "%s pre-pass dW%d" % (tag, i))
    if i < n - 1:
      _check(fails, "backward", c.dbs[i].cpu().numpy(), bw["db"][i], bw["db_b"][i], "%s pre-pass db%d" % (tag, i))
  names = [key + nm for i in range(n) for nm in ("w%d" % i, "b%d" % i)]
  grads = [c.dws[i].cpu().numpy() if j == 0 else (c.dbs[i].cpu().numpy() if i < n - 1 else g.sum(axis=0))
           for i in range(n) for j in (0, 1)]
  gerr = [None] * (2 * n - 1) + [TOL * np.abs(g).sum(axis=0) + gb.sum(axis=0)]
  check_update(fails, spec["opt"], [pre[nm] for nm in names], grads, pre, post, key + "sub_opt_", names,
               tag + " pre-pass", grad_err=gerr)
  check_planes_resplit(fails, [("W%d" % i, w, wp) for i, (w, wp) in enumerate(zip(c.net.ws, c.net.wps))], tag)
  _, _, _, main_logits = check_forward(fails, case, c, spec, post, x, step_dev, floor_x, tag + " main pass")
  check_heads(fails, case, c, main_logits, y, tag + " main pass")


def _head_key(plan, gidx, h):
  for c in plan.candidates:
    if c.ehead is h:
      return "c%d_" % c.index
  return "h%d_" % gidx


def _members(case, plan, fnets, gidx, h):
  """the nets candidate ensemble `gidx` must read, from the case description (not from the head itself): the kept
  frozen members, then the new subnetworks it names (GrowStrategy: every frozen member and its own candidate)"""
  from adanet_b200.core import engine as eng
  by_index = {c.index: c.net for c in plan.candidates}      # a rank of a multi-rank search holds some candidates only
  if case.get("heads"):
    _, builders, keep, _ = case["heads"][gidx]
    return [fnets[i] for i in eng.kept_indices(keep, len(fnets))] + [by_index[b] for b in builders]
  return list(fnets) + [by_index[gidx]]


def check_head(fails, case, plan, fnets, gidx, h, pre, post, x, y, step_dev, cap, tag, planes, f16):
  """one candidate ensemble over the engine's member values: out3, mixture-weight / bias gradients (MATRIX: its own
  GEMMs mw_logits, the L1 norms mw_l1, dens and d_mw), the update, the EMA and trace row"""
  from adanet_b200 import _lib
  key = _head_key(plan, gidx, h)
  members = _members(case, plan, fnets, gidx, h)
  ens = h.ens
  floor_x = F16_FLOOR if f16 else 0.0
  gam = [float(v) for v in h.gammas]
  train = h.ens_opt is not None
  use_bias = bool(ens.use_bias) and train
  if h.mix == _lib.MIX_MATRIX:
    N, C = len(members), h.C
    lasts = [(_merge(m.hp[-1], m.batch, m.dims[-2]) if len(m.dims) > 2 else f64(x)) for m in members]
    Ws = [f64(pre[key + "mix%d" % k]) for k in range(N)]
    mwl = []
    for k in range(N):
      ex, bd = layer_fwd(lasts[k], Ws[k], np.zeros(C), False, floor=floor_x)
      got = h.mw_logits[k].cpu().numpy()
      _check(fails, "heads", got, ex, bd, "%s mw_logits %d" % (tag, k))
      mwl.append(f64(got))
    l1 = np.array([np.abs(W).sum() for W in Ws])
    _check(fails, "heads", h.mw_l1.cpu().numpy(), l1, 2 * U * np.array([W.size for W in Ws]) * l1, tag + " mw_l1")
    bias = f64(pre[key + "bias"])
    e = bias + sum(mwl)
    e_err = 2 * (N + 1) * U * (np.abs(bias) + sum(np.abs(m) for m in mwl))
    loss, lb, g, gb = head_loss(case["head"], e, y, e_err)
    reg_on = not h.reg_is_zero
    reg = float(sum(gm * v for gm, v in zip(gam, l1))) if reg_on else 0.0
    reg_b = 2 * (sum(W.size for W in Ws) + N) * U * reg
    out3 = np.array([loss, reg, loss + reg])
    _check(fails, "heads", h.out3.cpu().numpy(), out3, np.array([lb, reg_b, lb + reg_b]) + 4 * U * np.abs(out3), tag + " out3")
    names, grads = [], []
    if train:
      dens = f64(h.dens.cpu().numpy())
      _check(fails, "heads", dens, g, gb, tag + " dens")
      floor_g = F16_FLOOR * 2.0 ** -h.dz_log2 if f16 else 0.0
      for k in range(N):
        L = np.abs(lasts[k])
        ex = lasts[k].T @ dens + (h.reg_multiplier * gam[k] * np.sign(Ws[k]) if reg_on else 0.0)
        bd = TOL * (L.T @ np.abs(dens)) + floor_g * L.sum(axis=0)[:, None] + floor_x * np.abs(dens).sum(axis=0)[None, :]
        bd = bd + 4 * U * h.reg_multiplier * abs(gam[k])
        _check(fails, "heads", h.d_mw[k].cpu().numpy(), ex, bd, "%s d_mw %d" % (tag, k))
      names = [key + "mix%d" % k for k in range(N)]
      grads = [t.cpu().numpy() for t in h.d_mw]
      d_bias_exact, d_bias_b = g.sum(axis=0), TOL * np.abs(g).sum(axis=0) + gb.sum(axis=0)
  else:
    mtype = "scalar" if h.mix == _lib.MIX_SCALAR else "vector"
    eh = ensemble(case["head"], mtype, pre[key + "mix0"], pre[key + "bias"], [m.logits.cpu().numpy() for m in members],
                  y, gam, h.reg_multiplier, use_bias)
    _check(fails, "heads", h.out3.cpu().numpy(), eh["out3"], eh["out3_b"], tag + " out3")
    names, grads = [], []
    if train:
      _check(fails, "heads", h.d_mix_w.cpu().numpy(), eh["dmw"].reshape(h.d_mix_w.shape), eh["dmw_b"].reshape(h.d_mix_w.shape),
             tag + " d_mix_w")
      names, grads = [key + "mix0"], [h.d_mix_w.cpu().numpy()]
      if use_bias:
        d_bias_exact, d_bias_b = eh["db"], eh["db_b"]
  if use_bias:
    _check(fails, "heads", h.d_bias.cpu().numpy(), d_bias_exact, d_bias_b, tag + " d_bias")
    names, grads = names + [key + "bias"], grads + [h.d_bias.cpu().numpy()]
  mix_keys = [kk for kk in pre if kk.startswith(key + "mix")] + [key + "bias"]
  if train:
    check_update(fails, ens.optimizer, [pre[nm] for nm in names], grads, pre, post, key + "ens_opt_", names, tag + " ensemble")
    if h.mix == _lib.MIX_MATRIX:
      check_planes_resplit(fails, [("mixture weight %d" % k, w, wp) for k, (w, wp) in enumerate(zip(h.mw, h.mwp))], tag)
  for kk in mix_keys:
    if kk not in names and not np.array_equal(pre[kk], post[kk]):
      fails.append("%s: %s changed, though nothing trains it" % (tag, kk))
  check_bookkeeping(fails, h, pre, post, key, step_dev, float(h._sub_loss_src[0].item()), cap, tag)


def teacher_forced_step(plan, fnets, case, frozen, cands, k, fails, inject=None, trace_capacity=4096):
  """one step of the plan, every stage against float64"""
  import torch
  from adanet_b200 import _lib
  planes = plan.xp is not None
  f16 = planes and _lib.plane_format() == _lib.PLANES_F16
  _FMT[0] = ("f16" if f16 else "tf32") if planes else "simt"
  if inject is not None:
    st = plan.state_dict()
    inject(plan, st, np.random.default_rng(77 + k), k)
    plan.load_state_dict(st)
  pre = plan.state_dict()
  step_dev = int(pre["step_dev"])
  frozen_before = _frozen_snapshot(fnets)
  x, y = _batch(case, k)
  own = {c.index: _batch(case, 500 + k) for c in plan.candidates if c.bagged}
  plan.train_step(x, y, own_batches=own or None)
  torch.cuda.synchronize()
  post = plan.state_dict()
  tag0 = "step %d" % (k + 1)
  check_frozen_forward(fails, fnets, frozen, x, F16_FLOOR if f16 else 0.0, planes)
  for c, spec in zip(plan.candidates, cands):
    tag = "%s cand %d" % (tag0, c.index)
    if c.bagged:
      check_bagged(fails, case, c, spec, pre, post, own[c.index], x, y, step_dev, tag, f16)
    else:
      check_candidate(fails, case, c, spec, pre, post, x, y, step_dev, tag, planes, f16)
  for gidx, h, _ in plan.heads:
    check_head(fails, case, plan, fnets, gidx, h, pre, post, x, y, step_dev, trace_capacity, "%s head %s" % (tag0, h.name), planes, f16)
  if int(post["step_dev"]) != step_dev + 1:
    fails.append("%s: step_dev %d -> %d" % (tag0, step_dev, int(post["step_dev"])))
  for j, (f, snap) in enumerate(zip(fnets, frozen_before)):
    for a, b in zip(f.ws + f.bs + (f.wps or []), snap):
      if not torch.equal(a.view(torch.int32), b.view(torch.int32)):
        fails.append("%s: frozen member %d changed" % (tag0, j))
        break
  return pre, post


def _run_steps(case, name, label):
  from adanet_b200 import _lib
  frozen, cands, warm = _case_data(case, seed=11)
  plan, fnets = _build_plan(case, frozen, cands, warm)
  fails = []
  for k in range(3):
    inject = case.get("inject") if k in (0, 2) else None
    teacher_forced_step(plan, fnets, case, frozen, cands, k, fails, inject)
    assert not fails, "%s (%s):\n%s" % (name, label, "\n".join(fails[:30]))
  return plan


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_CASES)
def test_teacher_forced_steps(fmt, name):
  """Three steps (eager, capture + replay, replay), each stage element-wise against float64."""
  from adanet_b200 import _lib
  plan = _run_steps(CASES[name], name, fmt + " planes")
  assert plan._graph is not None
  assert not _lib.plane_overflow()


@pytest.fixture(scope="module")
def simt_path():
  from tests.test_gpu_plane_groups import _open
  _, _lib, _ = _open()
  _lib.set_dense_path(_lib.PATH_SIMT)
  yield
  _lib.set_dense_path(_lib.PATH_AUTO)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SIMT_CASES)
def test_teacher_forced_steps_simt(simt_path, name):
  """The same steps on the fp32 CUDA-core cross-check path (adn_set_dense_path(SIMT)): every candidate runs its whole
  step on its own stream (IterationPlan._enqueue), dense fp32 activations and gradients, every GEMM entry within the
  classical fp32 dot-product bound (K + 2) U."""
  plan = _run_steps(CASES[name], name, "simt")
  assert plan.xp is None and plan.multi_stream == (len(plan.candidates) > 1)
  assert plan._graph is not None


@pytest.mark.gpu
def test_trace_wrap_and_eval(fmt):
  """trace_capacity = 5 over 7 steps: traces() holds the last 5 steps' rows, oldest first.  Then eval_step from the
  trained state: adanet_loss and accuracy of every head against float64 of the members' forward without dropout, and
  the training state byte-identical after it."""
  import torch
  case = dict(CASES["dropout"], inject=None)
  frozen, cands, warm = _case_data(case, seed=13)
  plan, fnets = _build_plan(case, frozen, cands, warm, trace_capacity=5)
  fails, rows = [], []
  for k in range(7):
    pre, post = teacher_forced_step(plan, fnets, case, frozen, cands, k, fails, trace_capacity=5)
    rows.append({h.name: post["c%d_trace" % h_i][k % 5].copy() for h_i, (_, h, _) in enumerate(plan.heads)})
    assert not fails, "\n".join(fails[:30])
  tr = plan.traces()
  for h_i, (_, h, _) in enumerate(plan.heads):
    want = np.stack([r[h.name] for r in rows[2:]])
    got = np.stack([tr[h.name][f] for f in ("sub_loss", "ens_loss", "adanet_loss", "ema")], axis=1)
    assert np.array_equal(got, want), "traces() of %s after 7 steps in a ring of 5:\n%s\nwant\n%s" % (h.name, got, want)
  # evaluation
  before = plan.state_dict()
  xe, ye = _batch(case, 99)
  losses = plan.eval_step(xe, ye, "adanet_loss")
  acc = plan.eval_step(xe, ye, "accuracy")
  after = plan.state_dict()
  for key in before:
    assert np.array_equal(before[key], after[key], equal_nan=True), "eval_step changed %s" % key
  f_logits = []
  for f in frozen:
    h = f64(xe)
    for i, (w, b) in enumerate(zip(*f["p"])):
      h, _ = layer_fwd(h, w, b, i < len(f["p"][0]) - 1)
    f_logits.append(h)
  for j, c in enumerate(plan.candidates):
    key = "c%d_" % c.index
    h = f64(xe)
    for i in range(len(c.net.ws)):
      h, _ = layer_fwd(h, before[key + "w%d" % i], before[key + "b%d" % i], i < len(c.net.ws) - 1)
    eh = ensemble(case["head"], "scalar", before[key + "mix0"], before[key + "bias"], f_logits + [h], ye,
                  [float(v) for v in c.ehead.gammas], c.ehead.reg_multiplier, False)
    want = eh["out3"][2]
    assert abs(losses[j] - want) <= 1e-5 * max(1.0, abs(want)), "eval adanet_loss of %s: %r, want %r" % (c.ehead.name, losses[j], want)
    pred = eh["e"].argmax(axis=1)
    margin = np.sort(eh["e"], axis=1)
    clear = (margin[:, -1] - margin[:, -2]) > 1e-4
    assert abs(acc[j] - float((pred == ye).mean())) <= (~clear).sum() / len(ye) + 1e-7, "eval accuracy of %s" % c.ehead.name


# ------------------------------------------------------------------------------------------------------------------
# row-sharded candidate with dropout on two ranks
# ------------------------------------------------------------------------------------------------------------------
SHARD_CASE = dict(B=256, C=10, head="softmax_xent", frozen=[[D, 10]],
                  cands=[dict(dims=[D, 96, 64, 10], opt=("momentum", 0.02, 0.9), dropout=[(0.25, 7), (0.5, 9)])],
                  ens=dict(ENS, use_bias=True), inject=_inject_step(2 ** 32 + 3))


def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return s.getsockname()[1]


def _shard_worker(rank, world, port, fmt_name, q):
  import torch
  import torch.distributed as dist
  os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
  if torch.cuda.device_count() >= world:
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  else:        # fewer GPUs than ranks: share cuda:0, exchange over gloo
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    from tests.test_gpu_plane_groups import _open, _set_format
    from adanet_b200.core import engine as eng
    _, _lib, _ = _open()
    _set_format(_lib, fmt_name)
    case = SHARD_CASE
    frozen, cands, warm = _case_data(case, seed=17)
    comm = eng.ShardComm([0, 1], rank, None)
    plan, fnets = _build_plan(case, frozen, cands, warm, shards={0: comm})
    c = plan.candidates[0]
    out = []
    for k in range(2):
      st = plan.state_dict()
      case["inject"](plan, st, None, k)
      plan.load_state_dict(st)
      pre = plan.state_dict()
      x, y = _batch(case, k)
      plan.train_step(x, y)
      torch.cuda.synchronize()
      post = plan.state_dict()
      hs, logits = _engine_fwd(c, c.batch, x[c.row0:c.row0 + c.batch])
      out.append(dict(pre=pre, post=post, hs=hs, logits=logits, dl=c.dlogits.cpu().numpy(), row0=c.row0,
                      dws=[t.cpu().numpy() for t in c.dws], dbs=[t.cpu().numpy() for t in c.dbs],
                      sub_out3=c.sub_out3.cpu().numpy(), out3=c.ehead.out3.cpu().numpy(),
                      d_mix_w=c.ehead.d_mix_w.cpu().numpy(), d_bias=c.ehead.d_bias.cpu().numpy(),
                      f_logits=[f.logits.cpu().numpy() for f in fnets], f16=_lib.plane_format() == _lib.PLANES_F16,
                      dz_log2=c.dz_log2))
    q.put((rank, out))
  finally:
    dist.destroy_process_group()


@pytest.mark.gpu
def test_row_sharded_dropout_step(fmt):
  """A dropout candidate row-sharded over two ranks (two processes sharing cuda:0 over gloo, or NCCL on two GPUs),
  step_dev past 2^32.  Each rank's hidden layers carry ITS rows of the whole minibatch's mask; the averaged gradients
  and the next state equal the full-batch float64 step; the two ranks' states are byte-identical."""
  import torch.multiprocessing as mp
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, fmt, q)) for r in range(2)]
  for p in procs:
    p.start()
  got = {}
  for _ in procs:
    rank, out = q.get(timeout=300)
    got[rank] = out
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  case = SHARD_CASE
  frozen, cands, _ = _case_data(case, seed=17)
  spec = cands[0]
  fails = []
  for k in range(2):
    r0, r1 = got[0][k], got[1][k]
    for key in r0["post"]:
      if key != "steps_done" and not np.array_equal(r0["post"][key], r1["post"][key], equal_nan=True):
        fails.append("step %d: the ranks' %s differ" % (k + 1, key))
    pre, post = r0["pre"], r0["post"]
    step_dev = int(pre["step_dev"])
    x, y = _batch(case, k)
    B = case["B"]
    floor_x = F16_FLOOR if r0["f16"] else 0.0
    n = len(spec["dims"]) - 1
    hs_full, masks, muls = [], [], []
    for r in (r0, r1):
      tag = "step %d rank %d" % (k + 1, 0 if r is r0 else 1)
      Bl = B // 2
      for i in range(n):
        w, b = pre["c0_w%d" % i], pre["c0_b%d" % i]
        last = i == n - 1
        d = spec["dropout"][i] if not last else None
        keep = orc.dropout_keep_mask(d[1], i, step_dev, B, w.shape[1], d[0])[r["row0"]:r["row0"] + Bl] if d else None
        exact, bound = layer_fwd(r["hs"][i], w, b, not last, keep, d[0] if d else 0.0, floor_x)
        _check(fails, "forward", r["logits"] if last else r["hs"][i + 1], exact, bound, "%s layer %d" % (tag, i))
    # the averaged gradients = the full-batch ones: full dlogits = the local ones (local means) / 2, stacked
    hs_full = [np.concatenate([r0["hs"][i], r1["hs"][i]]) for i in range(n)]
    masks = [None] + [hs_full[i] > 0 for i in range(1, n)]
    muls = [1.0] + [1.0 / (1.0 - float(np.float32(spec["dropout"][i - 1][0]))) for i in range(1, n)]
    dl = np.concatenate([r0["dl"], r1["dl"]]).astype(np.float64) / 2
    loss, lb, g, gb = head_loss(case["head"], np.concatenate([r0["logits"], r1["logits"]]), y)
    _check(fails, "heads", dl, g, gb, "step %d full dlogits" % (k + 1))
    _check(fails, "heads", r0["sub_out3"][:1], loss, lb, "step %d sub_loss (averaged)" % (k + 1))
    floor_g = F16_FLOOR * 2.0 ** -r0["dz_log2"] if r0["f16"] else 0.0
    ws = [pre["c0_w%d" % i] for i in range(n)]
    bw = backward(ws, hs_full, dl, masks, muls, floor_g, floor_x)
    for i in range(n):
      _check(fails, "backward", r0["dws"][i], bw["dw"][i], bw["dw_b"][i], "step %d averaged dW%d" % (k + 1, i))
      if i < n - 1:
        _check(fails, "backward", r0["dbs"][i], bw["db"][i], bw["db_b"][i], "step %d averaged db%d" % (k + 1, i))
    members = [np.concatenate([r0["f_logits"][0][r0["row0"]:r0["row0"] + B // 2], r1["f_logits"][0][r1["row0"]:r1["row0"] + B // 2]]),
               np.concatenate([r0["logits"], r1["logits"]])]
    gam = _gammas(case["ens"], [f["cx"] for f in frozen] + [spec["cx"]])
    eh = ensemble(case["head"], "scalar", pre["c0_mix0"], pre["c0_bias"], members, y, gam, 2.0, True)
    _check(fails, "heads", r0["out3"], eh["out3"], eh["out3_b"], "step %d out3 (averaged)" % (k + 1))
    _check(fails, "heads", r0["d_mix_w"], eh["dmw"], eh["dmw_b"], "step %d d_mix_w (averaged)" % (k + 1))
    _check(fails, "heads", r0["d_bias"], eh["db"], eh["db_b"], "step %d d_bias (averaged)" % (k + 1))
    names = ["c0_" + nm for i in range(n) for nm in ("w%d" % i, "b%d" % i)]
    grads = [a for i in range(n) for a in (r0["dws"][i], r0["dbs"][i])]
    check_update(fails, spec["opt"], [pre[nm] for nm in names], grads, pre, post, "c0_sub_opt_", names, "step %d" % (k + 1))
    if int(post["step_dev"]) != step_dev + 1:
      fails.append("step %d: step_dev" % (k + 1))
  assert not fails, "\n".join(fails[:30])
