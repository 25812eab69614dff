"""Search configurations whose heads are wider than the narrow head kernel takes (dim > 64, or more members x dim than
its shared-memory slab holds), shared by the host conditioning check and the GPU parity tests of the wide head
kernel.  Same form as tests/test_gpu_iteration.CONFIGS."""

import numpy as np

from tests import parity_util as pu
from tests.parity_util import orc

ENS = dict(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001)

CONFIGS = {
    # research/improve_nas trains 100-class heads (cifar100.py:153-155)
    "c100_scalar": dict(data=("tabular", 4096, 100, 100, 101), cfgs=[(1, 64), (2, 64)], B=256, steps=20, iters=2,
                        opt=("sgd", 0.05), ens=ENS),
    "c100_vector_bias": dict(data=("tabular", 4096, 100, 100, 102), cfgs=[(1, 64), (2, 48)], B=256, steps=20, iters=2,
                             opt=("sgd", 0.05),
                             ens=dict(optimizer=("sgd", 0.05), adanet_lambda=0.01, adanet_beta=0.001, use_bias=True,
                                      mixture_weight_type="vector")),
    "c100_matrix": dict(data=("tabular", 4096, 100, 100, 103), cfgs=[(1, 64), (2, 48)], B=256, steps=15, iters=2,
                        opt=("sgd", 0.05),
                        ens=dict(optimizer=("sgd", 0.02), adanet_lambda=0.01, adanet_beta=0.001, use_bias=True,
                                 mixture_weight_type="matrix")),
    "c1000_small_batch": dict(data=("tabular", 1024, 50, 1000, 104), cfgs=[(1, 32), (2, 32)], B=48, steps=10, iters=2,
                              opt=("sgd", 0.1), ens=ENS),
    # RegressionHead(label_dimension=96)
    "regression96": dict(data=("regression_wide", 2048, 20, 96, 105), cfgs=[(1, 32), (2, 32)], B=128, steps=20, iters=2,
                         opt=("sgd", 0.05), ens=ENS, head="mse"),
    # 48 classes: the ensemble head holds one more member every iteration and leaves the narrow kernel (whose slab
    # fits 8 members at dim 48) at iteration 8, while the subnetwork losses stay on it
    "c48_force_grow": dict(data=("tabular", 4096, 30, 48, 106), cfgs=[(1, 16), (1, 24)], B=128, steps=4, iters=10,
                           opt=("sgd", 0.05), ens=ENS, force_grow=True),
}


def data(kind, n, d, c, seed):
  if kind == "tabular":
    return orc.make_tabular(n, d, c, seed=seed)
  if kind == "regression_wide":
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)).astype(np.float32)
    t = rng.standard_normal((d, c)).astype(np.float32) * np.float32(0.2)
    y = (x @ t + 0.1 * rng.standard_normal((n, c))).astype(np.float32)
    return x, y
  raise ValueError(kind)


def oracle_run(cfg, perm=None):
  kind, n, d, c, seed = cfg["data"]
  x, y = data(kind, n, d, c, seed)
  if perm is not None:
    x = np.ascontiguousarray(x[:, perm])

  def space(t, frozen):
    specs = pu.make_specs(cfg["cfgs"], d, c, t, cfg["opt"])[0]
    if perm is not None:
      for s in specs:
        s.ws[0] = np.ascontiguousarray(s.ws[0][perm])
    return specs

  res, _ = orc.run_adanet(space, x, y, cfg["B"], cfg["steps"], cfg["iters"], orc.EnsemblerSpec(**cfg["ens"]), c,
                          head=cfg.get("head", "softmax_xent"), force_grow=cfg.get("force_grow", False))
  return res


def engine_run(cfg):
  from adanet_b200.core import engine as eng
  from adanet_b200.core import search as srch
  kind, n, d, c, seed = cfg["data"]
  x, y = data(kind, n, d, c, seed)
  space = lambda t, frozen: pu.make_specs(cfg["cfgs"], d, c, t, cfg["opt"])[1]
  s = srch.AdaNetSearch(space, eng.EnsemblerPlanSpec(**cfg["ens"]), d, c, cfg["B"], head=cfg.get("head", "softmax_xent"),
                        force_grow=cfg.get("force_grow", False))
  reps = s.run(srch.consecutive_batches(x, y, cfg["B"]), cfg["steps"], cfg["iters"])
  return reps, s
