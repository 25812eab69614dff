"""NumPy reference for subnetworks whose dense layers read a concat of pieces (SubnetworkPlanSpec.inputs): their own
previous layer (the input features for the first layer), the input features again, or hidden layers of
previous-iteration members.  Built on the primitives of oracle/adanet_oracle.py, whose plain-chain functions it
leaves as they are: a layer over pieces is y = act(sum_p x_p W[rows_p] + b), its dW the piece dWs stacked in concat
order, and only the primary piece receives dX.  Arithmetic runs in the dtype of the weights (fp64 in the checks)."""

from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle import adanet_oracle as orc


@dataclass
class ConnectedSpec(orc.SubnetworkSpec):
  inputs: Optional[list] = None


@dataclass
class ConnectedMember(orc.FrozenMember):
  inputs: Optional[list] = None


def _pieces(inputs, i: int, width: int) -> list:
  if inputs is not None and inputs[i]:
    return inputs[i]
  return [{"src": "own", "rows": [0, width]}]


def connected_forward(ws, bs, x, inputs, member_acts: Dict[Tuple[int, str], List[np.ndarray]], dropout=None):
  """(acts [x, h_1, ..., logits], piece inputs per layer).  `member_acts[(iteration, name)]`: that member's acts (its
  layer j is acts[j + 1]); `dropout` as in adanet_oracle.mlp_forward."""
  dt = np.asarray(ws[0]).dtype
  x = np.asarray(x, dtype=dt)
  acts, xs = [x], []
  n = len(ws)
  for i in range(n):
    px = []
    for p in _pieces(inputs, i, np.shape(ws[i])[0]):
      if p["src"] == "own":
        px.append(acts[-1])
      elif p["src"] == "input":
        px.append(x)
      else:
        px.append(np.asarray(member_acts[(p["iteration"], p["name"])][p["layer"] + 1], dtype=dt))
    xs.append(px)
    rows = [p["rows"] for p in _pieces(inputs, i, np.shape(ws[i])[0])]
    z = sum(a @ ws[i][r0:r1] for a, (r0, r1) in zip(px, rows)) + bs[i]
    if i < n - 1:
      z = np.maximum(z, 0)
      d = dropout[0][i] if (dropout is not None and dropout[0] is not None) else None
      if d is not None:
        keep = orc.dropout_keep_mask(d[1], i, dropout[1], z.shape[0], z.shape[1], d[0])
        z = np.where(keep, z * (1.0 / (1.0 - float(d[0]))), 0)
    acts.append(np.asarray(z, dtype=dt))
  return acts, xs


def connected_backward(ws, acts, xs, dlogits, inputs, dropout=None):
  """(dWs, dbs, dXs): dWs[i] = the piece dWs of layer i stacked in concat order (the kernel's gradient); dXs[i] = the
  gradient w.r.t. hidden layer i - 1 formed from the primary piece's rows (None for the first layer)."""
  n = len(ws)
  dws, dbs, dxs = [None] * n, [None] * n, [None] * n
  dz = np.asarray(dlogits, dtype=np.asarray(ws[0]).dtype)
  for i in range(n - 1, -1, -1):
    ps = _pieces(inputs, i, np.shape(ws[i])[0])
    dws[i] = np.concatenate([a.T @ dz for a in xs[i]], axis=0)
    dbs[i] = dz.sum(axis=0)
    if i > 0:
      r0, r1 = next(p["rows"] for p in ps if p["src"] == "own")
      dh = dz @ ws[i][r0:r1].T
      dxs[i] = dh
      d = dropout[0][i - 1] if (dropout is not None and dropout[0] is not None) else None
      if d is not None:
        dh = dh * (1.0 / (1.0 - float(d[0])))
      dz = dh * (acts[i] > 0)
  return dws, dbs, dxs


def _member_acts(frozen: Sequence[ConnectedMember], x):
  """Inference forwards of the frozen members in member order (a member reads only earlier ones)."""
  out = {}
  for f in frozen:
    out[(f.iteration, f.name)] = connected_forward(f.ws, f.bs, x, getattr(f, "inputs", None), out)[0]
  return out


def train_step(cands, frozen: Sequence[ConnectedMember], ens: orc.EnsemblerSpec, x, y, head: str = "softmax_xent"):
  """adanet_oracle.train_step (GrowStrategy, SCALAR / VECTOR, no bagging) for connected subnetworks."""
  head_fn = orc.HEADS[head]
  f32 = orc.F32
  macts = _member_acts(frozen, x)
  frozen_acts = [macts[(f.iteration, f.name)] for f in frozen]
  for c in cands:
    drop = (c.subnetwork.dropout, len(c.trace_sub_loss)) if c.subnetwork.dropout else None
    acts, xs = connected_forward(c.ws, c.bs, x, c.subnetwork.inputs, macts, drop)
    sub_loss, dlogits = head_fn(acts[-1], y)
    m_logits = [a[-1] for a in frozen_acts] + [acts[-1]]
    m_last = [a[-2] for a in frozen_acts] + [acts[-2]]
    e_logits = orc.ensemble_logits(ens.mixture_weight_type, c.weights, c.bias, m_logits, m_last)
    ens_loss, g = head_fn(e_logits, y)
    reg = orc.complexity_regularization(c.weights, c.complexities, ens.adanet_lambda, ens.adanet_beta)
    adanet_loss = f32(ens_loss + reg)
    dws, dbs, _ = connected_backward(c.ws, acts, xs, dlogits, c.subnetwork.inputs, drop)
    if c.ens_opt is not None:
      mult = 1.0 if ens.legacy_train_op else 2.0
      dmw, dbias = orc.ensemble_grads(ens.mixture_weight_type, c.weights, c.complexities, ens.adanet_lambda,
                                      ens.adanet_beta, mult, g, m_logits, m_last, ens.use_bias)
      params, grads = list(c.weights), list(dmw)
      if ens.use_bias:
        params.append(c.bias)
        grads.append(dbias)
      c.ens_opt.apply(params, grads)
    params, grads = [], []
    for w, b, dw, db in zip(c.ws, c.bs, dws, dbs):
      params += [w, b]
      grads += [dw.astype(f32), db.astype(f32)]
    c.sub_opt.apply(params, grads)
    ema = c.ema.update(adanet_loss)
    c.trace_sub_loss.append(float(sub_loss))
    c.trace_ens_loss.append(float(ens_loss))
    c.trace_adanet_loss.append(float(adanet_loss))
    c.trace_ema.append(float(ema))


def run_adanet(search_space, x_all, y_all, batch_size: int, steps_per_iteration: int, iterations: int,
               ens: orc.EnsemblerSpec, logits_dim: int, adanet_loss_decay: float = 0.9, head: str = "softmax_xent"):
  """adanet_oracle.run_adanet (GrowStrategy) over ConnectedSpec search spaces: frozen members carry their pieces."""
  frozen: List[ConnectedMember] = []
  prev_best_ema, prev_arch, results, cursor = None, [], [], 0
  n = x_all.shape[0]
  for t in range(iterations):
    specs = search_space(t, frozen)
    cands = orc.build_candidates(t, specs, frozen, ens, logits_dim, adanet_loss_decay,
                                 prev_weights=results[-1].mixture_weights if results else None,
                                 prev_bias=results[-1].bias if results else None)
    for _ in range(steps_per_iteration):
      if cursor + batch_size > n:
        cursor = 0
      train_step(cands, frozen, ens, x_all[cursor:cursor + batch_size], y_all[cursor:cursor + batch_size], head)
      cursor += batch_size
    names = [c.name for c in cands]
    emas = [c.trace_ema[-1] for c in cands]
    if t > 0:
      names, emas = ["previous_ensemble"] + names, [prev_best_ema] + emas
    best = orc.select_best(emas, t)
    traces = {c.name: {"sub_loss": c.trace_sub_loss, "ens_loss": c.trace_ens_loss,
                       "adanet_loss": c.trace_adanet_loss, "ema": c.trace_ema} for c in cands}
    if t > 0 and best == 0:
      arch, mw, bias = list(prev_arch), results[-1].mixture_weights, results[-1].bias
    else:
      w = cands[best - (1 if t > 0 else 0)]
      frozen = list(frozen) + [ConnectedMember(t, w.subnetwork.name, w.ws, w.bs, w.subnetwork.complexity,
                                               inputs=w.subnetwork.inputs)]
      arch = list(prev_arch) + [(t, w.subnetwork.name)]
      prev_best_ema = emas[best]
      mw, bias = w.weights, w.bias
    prev_arch = arch
    results.append(orc.IterationResult(t, names, [float(e) for e in emas], best, arch, traces, mw, bias))
  return results, frozen


def ensemble_logits(frozen: Sequence[ConnectedMember], mixture_type: str, weights, bias, x):
  """Inference logits of a finished ensemble of connected members (evaluate / predict)."""
  macts = _member_acts(frozen, x)
  acts = [macts[(f.iteration, f.name)] for f in frozen]
  return orc.ensemble_logits(mixture_type, weights, bias, [a[-1] for a in acts], [a[-2] for a in acts])
