"""Two-GPU parity (SURVEY.md section 8e): candidates sharded over ranks, NCCL only at the iteration boundary.

Every rank trains the subnetworks / candidate ensembles it owns; at the end of an iteration the EMA losses are
all-gathered and the winner's weights broadcast (distributed/exchange.py).  The result -- per-step losses of every
candidate, selected index, architecture, mixture weights -- must equal the single-process oracle's, whatever the
placement.  With 2 GPUs on the machine the two ranks use one GPU each over NCCL; on a one-GPU box
both ranks run on cuda:0 and the exchange goes over gloo (distributed/exchange._comm_device), so the placement, the
gathered selection and the winner broadcast are exercised either way.
"""

import os
import socket

import numpy as np
import pytest

from tests import parity_util as pu
from tests.parity_util import orc

TOL = 1e-5

CASES = {
    # four subnetworks of very different cost -> LPT placement puts the widest alone on one rank
    "grow_balanced": dict(cfgs=[(1, 48), (2, 32), (3, 24), (2, 96)], strategies=("grow",), placement="balanced"),
    "grow_round_robin": dict(cfgs=[(1, 48), (2, 32), (3, 24)], strategies=("grow",), placement="round_robin"),
    # Solo + Grow heads over the same subnetwork stay with it
    "solo_grow": dict(cfgs=[(1, 48), (2, 32), (3, 24)], strategies=("solo", "grow"), placement="balanced"),
    # AllStrategy reads every subnetwork: one component, one rank; the other rank owns nothing this iteration
    "all_solo_grow": dict(cfgs=[(1, 48), (2, 32)], strategies=("all", "solo", "grow"), placement="balanced"),
    # a single candidate on two GPUs: rank 1 idles and still takes part in the exchange
    "one_candidate": dict(cfgs=[(2, 32)], strategies=("grow",), placement="balanced"),
    # row-sharded placement (distributed/exchange.sharded_placement): the wide candidate is 90 % of the work, so both
    # ranks train it data-parallel on half of the minibatch rows each and average its gradient arena every step; the
    # narrow ones stay whole.  Same per-step losses, selection and frozen weights as the single-process oracle.
    "sharded_rows": dict(cfgs=[(2, 160), (1, 16), (2, 24)], strategies=("grow",), placement="sharded"),
    # conv-stem subnetworks: the winner's stem kernel / bias travel in the end-of-iteration broadcast too
    "simple_cnn": dict(cnn=True),
}
# BASELINE config 4 in small: simple_cnn subnetworks (conv stem + dense) sharded over the two GPUs
CNN_CASE = dict(image=(16, 16, 3), seeds=(0, 1, 2, 3), filters=16, hidden=32, B=64, steps=8, iters=2)
D, C, B, STEPS, ITERS = 100, 10, 256, 12, 3
ENS = dict(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001, use_bias=True)


def _cnn_data():
  h, w, c = CNN_CASE["image"]
  rng = np.random.default_rng(3234)
  return (rng.uniform(0, 1, (512, h, w, c)) * 2 - 1).astype(np.float32), rng.integers(0, C, 512)


def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return s.getsockname()[1]


def _worker(rank, world, port, case, q):
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
    from adanet_b200.core import engine as eng
    from adanet_b200.core import search as srch
    if case.get("cnn"):
      cc = CNN_CASE
      x, y = _cnn_data()
      opt = ("momentum_cosine", 0.003, 0.9, cc["steps"])
      s = srch.AdaNetSearch(lambda t, frozen: pu.make_cnn_specs(cc["seeds"], cc["image"], cc["filters"], cc["hidden"], C, t, opt)[1],
                            eng.EnsemblerPlanSpec(), int(np.prod(cc["image"])), C, cc["B"], adanet_loss_decay=0.99)
      reps = s.run(srch.consecutive_batches(x, y, cc["B"]), cc["steps"], cc["iters"])
    else:
      x, y = orc.make_tabular(8192, D, C, seed=21)
      s = srch.AdaNetSearch(lambda t, frozen: pu.make_specs(case["cfgs"], D, C, t, ("sgd", 0.02))[1],
                            eng.EnsemblerPlanSpec(**ENS), D, C, B, strategies=case["strategies"],
                            placement=case["placement"])
      reps = s.run(srch.consecutive_batches(x, y, B), STEPS, ITERS)
    out = []
    for r in reps:
      mw = r.mixture_weights
      out.append(dict(names=list(r.candidate_names), ema=[float(v) for v in r.ema_losses], best=int(r.best_index),
                      arch=list(r.architecture), mw=np.asarray(mw), bias=np.asarray(r.bias),
                      traces={k: {f: np.asarray(v[f]) for f in ("sub_loss", "adanet_loss", "ema")}
                              for k, v in (r.traces or {}).items()}))
    frozen = [m.numpy_params()[0] for m in s.frozen]      # kernels in layer order (a conv stem's first)
    q.put((rank, out, frozen))
  finally:
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_two_gpu_search_matches_oracle(built_lib, name):
  import torch
  import torch.multiprocessing as mp
  case = CASES[name]
  if case.get("cnn"):
    cc = CNN_CASE
    x, y = _cnn_data()
    opt = ("momentum_cosine", 0.003, 0.9, cc["steps"])
    want, o_frozen = orc.run_adanet(lambda t, frozen: pu.make_cnn_specs(cc["seeds"], cc["image"], cc["filters"], cc["hidden"], C, t, opt)[0],
                                    x, y, cc["B"], cc["steps"], cc["iters"], orc.EnsemblerSpec(), C, adanet_loss_decay=0.99)
  else:
    x, y = orc.make_tabular(8192, D, C, seed=21)
    want, o_frozen = orc.run_adanet_strategies(lambda t, frozen: pu.make_specs(case["cfgs"], D, C, t, ("sgd", 0.02))[0], x, y,
                                               B, STEPS, ITERS, orc.EnsemblerSpec(**ENS), C, strategies=case["strategies"])
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_worker, args=(r, 2, port, case, q)) for r in range(2)]
  for p in procs:
    p.start()
  got = {}
  for _ in procs:
    rank, out, frozen = q.get(timeout=240)
    got[rank] = (out, frozen)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  seen = set()
  for rank in (0, 1):
    out, frozen = got[rank]
    for t, (r, ro) in enumerate(zip(out, want)):
      # every rank reaches the same decision from the gathered losses
      assert r["names"] == ro.candidate_names and r["best"] == ro.best_index and r["arch"] == ro.architecture
      np.testing.assert_allclose(r["ema"], ro.ema_losses, atol=TOL)
      np.testing.assert_allclose(r["mw"], np.asarray(ro.mixture_weights), atol=TOL)
      np.testing.assert_allclose(r["bias"], np.asarray(ro.bias), atol=TOL)
      for cname, tr in r["traces"].items():          # the candidates this rank trained, step by step
        seen.add((t, cname))
        for f in ("sub_loss", "adanet_loss", "ema"):
          np.testing.assert_allclose(tr[f], np.asarray(ro.traces[cname][f], dtype=np.float64), atol=TOL, equal_nan=True)
    # the frozen members (winner weights broadcast from their owner) agree on both ranks and with the oracle
    assert len(frozen) == len(o_frozen)
    for ws, m in zip(frozen, o_frozen):
      for w, wo in zip(ws, m.ws):
        np.testing.assert_allclose(w, wo, atol=5e-5)
  assert seen == {(t, cname) for t, ro in enumerate(want) for cname in ro.traces}   # every candidate trained somewhere


def _estimator_worker(rank, world, port, model_dir, placement, q):
  """adanet_b200.Estimator.train under a 2-rank job: what `torchrun` starts (RANK / WORLD_SIZE in the environment)."""
  import torch
  import torch.distributed as dist
  os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
  os.environ["RANK"], os.environ["WORLD_SIZE"] = str(rank), str(world)
  if torch.cuda.device_count() >= world:
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
  else:
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
  try:
    import adanet_b200 as adanet
    from adanet_b200 import graph, train
    from adanet_b200.examples import simple_dnn
    from tests import test_gpu_api as api
    x, y = api._data(orc)
    gen = api._modern(simple_dnn.Generator(feature_columns=[graph.numeric_column("x", api.D)],
                                           optimizer=train.GradientDescentOptimizer(0.05), layer_size=16, seed=api.SEED))
    est = adanet.Estimator(
        head=adanet.heads.MultiClassHead(api.C), subnetwork_generator=gen, max_iteration_steps=12,
        ensemblers=[adanet.ensemble.ComplexityRegularizedEnsembler(optimizer=train.GradientDescentOptimizer(0.01),
                                                                   adanet_lambda=0.01, adanet_beta=0.001)],
        max_iterations=3, model_dir=model_dir, debug=True, candidate_placement=placement)
    assert est.config.num_worker_replicas == world and est.config.is_chief == (rank == 0)
    est.train(api._input_fn(x, y), max_steps=36)
    reps = est._search.reports
    xe, ye = api._data(orc, n=api.B * 2, seed=99)
    ev = est.evaluate(api._input_fn(xe, ye), steps=2)
    q.put((rank, [dict(best=int(r.best_index), arch=list(r.architecture), ema=[float(v) for v in r.ema_losses],
                       traces={k: {f: np.asarray(v[f]) for f in ("sub_loss", "adanet_loss")} for k, v in r.traces.items()})
                  for r in reps], float(ev["loss"]), est.architecture_string()))
  finally:
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("placement", ["balanced", "sharded"])
def test_two_rank_estimator_matches_oracle(built_lib, tmp_path, placement):
  """The PUBLIC API under a multi-rank job (the chief/worker protocol of adanet/core/estimator.py:937-984 replaced by
  the end-of-iteration exchange): both ranks call Estimator.train with the same input_fn, each trains the candidates
  placed on it, and both end with the oracle's per-step losses, selections, architecture and evaluation loss; only
  the chief writes architecture-{t}.json."""
  import json
  import torch.multiprocessing as mp
  from tests import test_gpu_api as api
  x, y = api._data(orc)
  ens = orc.EnsemblerSpec(optimizer=("sgd", 0.01), adanet_lambda=0.01, adanet_beta=0.001)
  want, frozen = orc.run_adanet(api._oracle_simple_dnn_space(orc, 16, 0.05), x, y, api.B, 12, 3, ens, api.C)
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_estimator_worker, args=(r, 2, port, str(tmp_path), placement, q)) for r in range(2)]
  for p in procs:
    p.start()
  got = {}
  for _ in procs:
    rank, reps, ev_loss, arch = q.get(timeout=240)
    got[rank] = (reps, ev_loss, arch)
  for p in procs:
    p.join(timeout=60)
    assert p.exitcode == 0
  xe, ye = api._data(orc, n=api.B * 2, seed=99)
  want_eval = np.mean([api._oracle_eval(orc, frozen, want[-1].mixture_weights, want[-1].bias, xe[i:i + api.B], ye[i:i + api.B])[0]
                       for i in (0, api.B)])
  seen = set()
  for rank in (0, 1):
    reps, ev_loss, arch = got[rank]
    assert len(reps) == 3
    for t, (r, ro) in enumerate(zip(reps, want)):
      assert r["best"] == ro.best_index and r["arch"] == ro.architecture
      np.testing.assert_allclose(r["ema"], ro.ema_losses, atol=TOL)
      for cname, tr in r["traces"].items():
        seen.add((t, cname))
        for f in ("sub_loss", "adanet_loss"):
          np.testing.assert_allclose(tr[f], np.asarray(ro.traces[cname][f], dtype=np.float64), atol=TOL)
    assert abs(ev_loss - want_eval) < 1e-5
    assert arch == "| " + " | ".join(n for _, n in want[-1].architecture) + " |"
  assert seen == {(t, cname) for t, ro in enumerate(want) for cname in ro.traces}
  for t in range(3):
    a = json.load(open(os.path.join(str(tmp_path), "architecture-{}.json".format(t))))
    assert [s["builder_name"] for s in a["subnetworks"]] == [n for _, n in want[t].architecture]
