"""Generates tests/golden/*.json by importing the REFERENCE's own modules.

Needs a checkout of tensorflow/adanet v0.9.0 (the reference):
    python tests/golden/make_golden.py /path/to/adanet

The reference is a pure-Python TF1 library; TensorFlow is not installable
here, so only its TF-free modules can be executed:
  * adanet/distributed/placement.py  (with adanet.tf_compat stubbed -- only
    subnetwork_devices touches TF)
  * adanet/distributed/devices.py    (_OpNameHashStrategy: sha256 % ps)
  * adanet/ensemble/strategy.py
  * adanet/core/architecture.py
Known-answer vectors that live inside the reference's TF-dependent tests are
transcribed by hand into known_answers.json with their file:line.
"""

import importlib.util
import json
import os
import sys
import types

REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("ADANET_REFERENCE", "")
OUT = os.path.dirname(os.path.abspath(__file__))


def _load(name, path):
  spec = importlib.util.spec_from_file_location(name, path)
  mod = importlib.util.module_from_spec(spec)
  sys.modules[name] = mod
  spec.loader.exec_module(mod)
  return mod


def load_reference_modules():
  # Stub package skeleton so `from adanet import tf_compat` resolves.
  adanet = types.ModuleType("adanet")
  adanet.__path__ = []
  sys.modules["adanet"] = adanet
  tf_compat = types.ModuleType("adanet.tf_compat")
  sys.modules["adanet.tf_compat"] = tf_compat
  adanet.tf_compat = tf_compat
  dist = types.ModuleType("adanet.distributed")
  dist.__path__ = []
  sys.modules["adanet.distributed"] = dist
  devices = _load("adanet.distributed.devices", REF + "/adanet/distributed/devices.py")
  placement = _load("adanet.distributed.placement", REF + "/adanet/distributed/placement.py")
  strategy = _load("ref_strategy", REF + "/adanet/ensemble/strategy.py")
  architecture = _load("ref_architecture", REF + "/adanet/core/architecture.py")
  return devices, placement, strategy, architecture


class _Config:
  def __init__(self, num_workers, worker_index, num_ps=0):
    self.num_worker_replicas = num_workers
    self.global_id_in_cluster = worker_index
    self.num_ps_replicas = num_ps


class _Builder:
  def __init__(self, name):
    self.name = name


def main():
  devices, placement, strategy, architecture = load_reference_modules()

  # ---- placement truth tables (placement.py:228-285) ----
  rows = []
  for drop in (False, True):
    for nw in range(1, 9):
      for ns in (1, 2, 3, 5, 8):
        for wi in range(nw):
          s = placement.RoundRobinStrategy(drop_remainder=drop)
          s.config = _Config(nw, wi)
          rows.append({
              "drop_remainder": drop, "num_workers": nw, "worker_index": wi, "num_subnetworks": ns,
              "build_ensemble": bool(s.should_build_ensemble(ns)),
              "build_subnetwork": [bool(s.should_build_subnetwork(ns, i)) for i in range(ns)],
              "train_subnetworks": bool(s.should_train_subnetworks(ns)),
          })
  rep = placement.ReplicationStrategy()
  rep.config = _Config(3, 1)
  replication = {"build_ensemble": rep.should_build_ensemble(3),
                 "build_subnetwork": [rep.should_build_subnetwork(3, i) for i in range(3)],
                 "train_subnetworks": rep.should_train_subnetworks(3)}
  with open(os.path.join(OUT, "placement.json"), "w") as f:
    json.dump({"source": "adanet/distributed/placement.py RoundRobinStrategy/ReplicationStrategy executed",
               "round_robin": rows, "replication": replication}, f)

  # ---- op-name hash strategy (devices.py:24-45) ----
  names = ["dense/kernel", "dense/bias", "adanet/iteration_0/subnetwork_t0_dnn/dense_1/kernel",
           "mixture_weight", "bias", "step", "global_step", "a", "b", "c"]

  class _Op:
    def __init__(self, name):
      self.name = name
  hashes = []
  for n_ps in (1, 2, 3, 5, 7):
    st = devices._OpNameHashStrategy(n_ps)
    hashes.append({"num_tasks": n_ps, "assign": {n: int(st(_Op(n))) for n in names}})
  with open(os.path.join(OUT, "op_name_hash.json"), "w") as f:
    json.dump({"source": "adanet/distributed/devices.py _OpNameHashStrategy executed", "cases": hashes}, f)

  # ---- strategies (strategy.py:79-117) ----
  cases = []
  for new, prev in ([["a"], []], [["a", "b"], []], [["a", "b"], ["p0"]], [["x", "y", "z"], ["p0", "p1"]]):
    nb = [_Builder(n) for n in new]
    pb = [_Builder(n) for n in prev]
    entry = {"new": new, "prev": prev}
    for cls_name in ("GrowStrategy", "AllStrategy", "SoloStrategy"):
      cands = getattr(strategy, cls_name)().generate_ensemble_candidates(nb, pb)
      entry[cls_name] = [{"name": c.name,
                          "subnetwork_builders": [b.name for b in c.subnetwork_builders],
                          "previous": [b.name for b in c.previous_ensemble_subnetwork_builders]}
                         for c in cands]
    cases.append(entry)
  with open(os.path.join(OUT, "strategy.json"), "w") as f:
    json.dump({"source": "adanet/ensemble/strategy.py executed", "cases": cases}, f)

  # ---- architecture serialisation (architecture.py:132-173) ----
  arch_cases = []
  for cand, ens, subs, replay, it, gs in (
      ("linear_grow", "complexity_regularized", [(0, "linear")], [0], 0, 100),
      ("2_layer_dnn_grow", "complexity_regularized", [(0, "linear"), (1, "1_layer_dnn"), (2, "2_layer_dnn")],
       [1, 2, 1], 2, 900),
      ("all", "mean", [(0, "a"), (0, "b"), (3, "c")], [], 3, 12345),
  ):
    a = architecture._Architecture(cand, ens, replay_indices=list(replay))
    for s in subs:
      a.add_subnetwork(*s)
    ser = a.serialize(it, gs)
    back = architecture._Architecture.deserialize(ser)
    arch_cases.append({"candidate": cand, "ensembler": ens, "subnetworks": subs, "replay_indices": replay,
                       "iteration": it, "global_step": gs, "serialized": ser,
                       "grouped": [[i, list(n)] for i, n in a.subnetworks_grouped_by_iteration],
                       "roundtrip_subnetworks": [list(s) for s in back.subnetworks],
                       "roundtrip_global_step": back.global_step})
  with open(os.path.join(OUT, "architecture.json"), "w") as f:
    json.dump({"source": "adanet/core/architecture.py executed", "cases": arch_cases}, f)

  # ---- hand-transcribed known answers from TF-dependent reference tests ----
  known = {
      "ema": {  # adanet/core/candidate_test.py:83-132
          "source": "adanet/core/candidate_test.py:83-132",
          "decay": 0.999, "losses": [1.0, 0.5, 0.25], "want": [1.0, 0.750, 0.583], "places": 3,
          "eval_mode_want": 0.0},
      "complexity_regularization": {  # adanet/ensemble/weighted_test.py:147-481 (complexity=2 per _build_subnetwork :137)
          "source": "adanet/ensemble/weighted_test.py:147-481",
          "cases": [
              {"name": "default", "n": 1, "lambda": 0.0, "beta": 0.0, "weights": [1.0], "want": 0.0,
               "norms": [1.0], "fractions": [1.0]},
              {"name": "one_previous_network", "n": 2, "lambda": 0.0, "beta": 0.0, "weights": [0.5, 0.5],
               "want": 0.0, "norms": [0.5, 0.5], "fractions": [0.5, 0.5]},
              {"name": "one_previous_network_with_lambda", "n": 2, "lambda": 0.1, "beta": 0.0,
               "weights": [0.5, 0.5], "want": 0.2, "norms": [0.5, 0.5], "fractions": [0.5, 0.5]},
              {"name": "all_previous_networks_with_lambda", "n": 3, "lambda": 0.1, "beta": 0.0,
               "weights": [1 / 3., 1 / 3., 1 / 3.], "want": 0.2, "norms": [1 / 3.] * 3, "fractions": [1 / 3.] * 3},
              {"name": "all_previous_networks_and_two_subnetworks", "n": 4, "lambda": 0.1, "beta": 0.0,
               "weights": [0.25] * 4, "want": 0.2, "norms": [0.25] * 4, "fractions": [0.25] * 4},
              {"name": "all_nets_with_warm_start", "n": 4, "lambda": 0.1, "beta": 0.0,
               "weights": [1.0, 1.0, 0.25, 0.25], "want": 0.5, "norms": [1.0, 1.0, 0.25, 0.25],
               "fractions": [0.4, 0.4, 0.1, 0.1]},
          ],
          "complexity": 2.0},
      "mixture_weight_sgd": {  # adanet/ensemble/weighted_test.py:588-627
          "source": "adanet/ensemble/weighted_test.py:588-627",
          "lr": 0.1, "w0": 0.0, "loss": "2*w", "want_w": -0.2},
      "simple_dnn_names": {  # adanet/examples/simple_dnn_test.py:54-81
          "source": "adanet/examples/simple_dnn_test.py:54-81",
          "initial_num_layers_0": {"names": ["linear", "1_layer_dnn"], "complexities": [0.0, 1.0]},
          "initial_num_layers_1": {"names": ["1_layer_dnn", "2_layer_dnn"], "complexities": [1.0, 1.414]}},
      "replay": {  # adanet/core/estimator_test.py:3235-3311
          "source": "adanet/core/estimator_test.py:3235-3311",
          "indices": [2, 3, 1]},
  }
  with open(os.path.join(OUT, "known_answers.json"), "w") as f:
    json.dump(known, f, indent=1)
  print("wrote golden fixtures to", OUT)


if __name__ == "__main__":
  main()
