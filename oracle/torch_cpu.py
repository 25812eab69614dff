"""TEST / BENCH INFRASTRUCTURE ONLY -- never imported by the product (adanet_b200/).

A second CPU restatement of one AdaNet training step (SURVEY.md section 3.3 steps 1-13) for the iteration-0,
GrowStrategy, SCALAR-mixture-weight, SGD case that BASELINE configs[2] / bench.py time, written on torch CPU
tensors so that the GEMMs run on oneDNN / MKL with every host core (`torch.set_num_threads`).  It exists because
NumPy/OpenBLAS is a weak CPU arm on a many-core host (round-1 VERDICT, weak #6); `bench.py` times both and keeps the
faster as `cpu_baseline` / `--impl reference`.  `tests/test_oracle_golden.py::test_torch_cpu_port_matches_numpy_oracle`
pins it to `oracle/adanet_oracle.py` (which in turn is pinned to the reference's known-answer tests).

Reference arithmetic restated (file:line in tensorflow/adanet v0.9.0):
  dense + ReLU stack and its gradients      adanet/examples/simple_dnn.py:61-110          [TF]
  mean sparse softmax cross-entropy head    adanet/core/ensemble_builder.py:571-583       [TF]
  w * logits, complexity penalty, adanet loss, mixture-weight gradient (penalty counted twice on the
  Ensembler.build_train_op path)            adanet/ensemble/weighted.py:400-454,545-617; ensemble_builder.py:416-426
  zero-debiased EMA                         adanet/core/candidate.py:117-129
"""

from __future__ import annotations

from typing import List, Sequence

import numpy as np
import torch


class Candidate:
  def __init__(self, ws: Sequence[np.ndarray], bs: Sequence[np.ndarray], complexity: float):
    self.ws = [torch.tensor(np.asarray(w, dtype=np.float32)) for w in ws]
    self.bs = [torch.tensor(np.asarray(b, dtype=np.float32)) for b in bs]
    self.complexity = float(complexity)
    self.w = torch.ones((), dtype=torch.float32)       # one member at iteration 0: 1/N = 1 (weighted.py:360-366)
    self.biased, self.n = 0.0, 0
    self.trace = []                                     # (sub_loss, ens_loss, adanet_loss, ema) per step


def _xent(logits: torch.Tensor, y: torch.Tensor):
  """mean sparse softmax-CE and dLoss/dlogits = (softmax - onehot) / B"""
  m = logits.max(dim=1, keepdim=True).values
  z = logits - m
  e = torch.exp(z)
  s = e.sum(dim=1, keepdim=True)
  b = logits.shape[0]
  loss = (torch.log(s).squeeze(1) - z.gather(1, y.view(-1, 1)).squeeze(1)).mean()
  g = e / s
  g[torch.arange(b), y] -= 1.0
  return loss, g / b


def train_step(cands: List[Candidate], x: torch.Tensor, y: torch.Tensor, lr: float, ens_lr: float, lam: float, beta: float,
               decay: float = 0.9):
  """Every candidate trains one step on the minibatch (x [B, D] fp32, y [B] int64)."""
  for c in cands:
    acts = [x]
    n = len(c.ws)
    for i in range(n):
      z = torch.addmm(c.bs[i], acts[-1], c.ws[i])
      acts.append(torch.relu_(z) if i < n - 1 else z)
    logits = acts[-1]
    sub_loss, dz = _xent(logits, y)
    # candidate ensemble over its single member (pre-update values)
    ens_loss, g = _xent(c.w * logits, y)
    gamma = np.float32(beta) if lam == 0.0 else np.float32(np.float32(lam) * np.float32(c.complexity) + np.float32(beta))
    reg = float(gamma) * float(c.w.abs()) if (lam != 0.0 or beta != 0.0) else 0.0
    adanet = np.float32(np.float32(ens_loss) + np.float32(reg))
    dw_mix = (g * logits).sum() + 2.0 * float(gamma) * torch.sign(c.w)
    # backward through the subnetwork's own variables
    dws, dbs = [], []
    for i in range(n - 1, -1, -1):
      dws.append(acts[i].t().mm(dz))
      dbs.append(dz.sum(dim=0))
      if i > 0:
        dz = dz.mm(c.ws[i].t()) * (acts[i] > 0)
    dws.reverse()
    dbs.reverse()
    c.w = c.w - ens_lr * dw_mix
    for i in range(n):
      c.ws[i].sub_(dws[i], alpha=lr)
      c.bs[i].sub_(dbs[i], alpha=lr)
    # zero-debiased EMA [TF assign_moving_average(zero_debias=True)]
    c.biased = np.float32(c.biased - np.float32(np.float32(c.biased) - adanet) * np.float32(1.0 - decay))
    c.n += 1
    ema = np.float32(c.biased / np.float32(1.0 - np.float32(decay) ** c.n))
    c.trace.append((float(sub_loss), float(ens_loss), float(adanet), float(ema)))
