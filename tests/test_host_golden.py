"""Host-side mirror of the reference interface vs fixtures produced by executing
the reference's own modules (tests/golden/make_golden.py).  CPU only."""

import json
import os
import re

import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
  with open(os.path.join(GOLD, name)) as f:
    return json.load(f)


def test_round_robin_truth_tables():
  # adanet/distributed/placement_test.py:66-298 (truth tables), generated from the reference class itself
  from adanet_b200.distributed import ClusterConfig, RoundRobinStrategy
  rows = _load("placement.json")["round_robin"]
  assert len(rows) > 300
  for row in rows:
    s = RoundRobinStrategy(drop_remainder=row["drop_remainder"])
    s.config = ClusterConfig(row["num_workers"], row["worker_index"])
    ns = row["num_subnetworks"]
    assert s.should_build_ensemble(ns) == row["build_ensemble"], row
    assert [s.should_build_subnetwork(ns, i) for i in range(ns)] == row["build_subnetwork"], row
    assert s.should_train_subnetworks(ns) == row["train_subnetworks"], row


def test_replication_strategy():
  from adanet_b200.distributed import ClusterConfig, ReplicationStrategy
  want = _load("placement.json")["replication"]
  s = ReplicationStrategy()
  s.config = ClusterConfig(3, 1)
  assert s.should_build_ensemble(3) == want["build_ensemble"]
  assert [s.should_build_subnetwork(3, i) for i in range(3)] == want["build_subnetwork"]
  assert s.should_train_subnetworks(3) == want["train_subnetworks"]


def test_reference_round_robin_8_workers_8_subnetworks_finding():
  # SURVEY.md section 0 finding 2: worker0 -> ensemble only, worker1 -> subnets [0,7], workers 2-7 -> [1]..[6]
  from adanet_b200.distributed import ClusterConfig, RoundRobinStrategy
  got = []
  for wi in range(8):
    s = RoundRobinStrategy()
    s.config = ClusterConfig(8, wi)
    got.append([i for i in range(8) if s.should_build_subnetwork(8, i)] if s.should_train_subnetworks(8) else "ens")
  assert got == ["ens", [0, 7], [1], [2], [3], [4], [5], [6]]


def test_colocated_strategy_is_i_mod_g():
  from adanet_b200.distributed import ClusterConfig, ColocatedStrategy
  for g in (1, 2, 4, 8):
    seen = []
    for r in range(g):
      s = ColocatedStrategy()
      s.config = ClusterConfig(g, r)
      own = s.owned(32)
      assert all(i % g == r for i in own)
      assert s.should_train_subnetworks(32) and s.should_build_ensemble(32)
      seen += own
    assert sorted(seen) == list(range(32))


def test_cabi_header_symbols_are_exported(built_lib):
  """The shared library loads and exports every entry point include/adanet_b200.h declares."""
  from adanet_b200 import _lib
  hdr = open(os.path.join(ROOT, "include", "adanet_b200.h")).read()
  declared = sorted(set(re.findall(r"\b(adn_[a-z0-9_]+)\s*\(", hdr)))
  assert len(declared) >= 12
  for name in declared:
    assert hasattr(built_lib, name), "missing export %s" % name
  assert sorted(_lib.EXPORTS) == declared
  assert _lib.query(_lib.Q_VERSION) == 100


def test_cabi_argument_validation_without_gpu(built_lib):
  """Error behaviour of the boundary: bad arguments fail loudly with a message, before any launch."""
  from adanet_b200 import _lib
  rc = built_lib.adn_dense_fwd(None, None, None, None, 4, 4, 4, 0, None, 0, None)
  assert rc == -22 and b"null" in built_lib.adn_last_error()
  rc = built_lib.adn_dense_fwd(8, 8, None, 8, 0, 4, 4, 0, None, 0, None)
  assert rc == -22
  rc = built_lib.adn_dense_fwd(8, 8, None, 8, 4, 4, 4, 7, None, 0, None)
  assert rc == -22 and b"act" in built_lib.adn_last_error()
  rc = built_lib.adn_ema_update(None, None, 0.9, None)
  assert rc == -22
  with pytest.raises(_lib.AdnError):
    _lib.check(built_lib.adn_set_dense_path(9), "adn_set_dense_path")
  assert _lib.query(_lib.Q_DENSE_BWD_WS, 4096, 100, 1024) > 0
  assert _lib.query(_lib.Q_HEAD_WS, 4096, 10, 5) > 0
  _check_head_and_plane_validation(built_lib)


def _check_head_and_plane_validation(lib):
  """Every check of the head, colsum and plane-GEMM entry points rejects its call with the right code and a message
  naming the called function, before any launch: the pointers below are never dereferenced."""
  import ctypes
  from adanet_b200 import _lib
  INVALID, UNSUPPORTED, WORKSPACE = -22, -95, -12
  P, BIG = 1 << 20, 1 << 40           # fake device pointer / workspace size
  members = _lib.ptr_array([P + 256 * k for k in range(64)])
  gam = _lib.f32_array([0.5] * 64)
  before = _lib.launch_count()

  def rejects(name, want, phrase, *args):
    rc = getattr(lib, name)(*args)
    msg = lib.adn_last_error().decode()
    assert (rc, phrase in msg, name in msg) == (want, True, True), (name, phrase, rc, msg)

  def ens_head(want, phrase, **kw):
    a = dict(head=0, mix=0, members=members, n=2, w=P, bias=None, gammas=gam, reg_is_zero=0, mult=1.0, labels=P,
             labels_f=None, out3=P, dw=None, dbias=None, dens=None, ens_out=None, batch=256, dim=10, ws=P, ws_bytes=BIG)
    a.update(kw)
    rejects("adn_ensemble_head", want, phrase, *a.values(), None)

  ens_head(INVALID, "null pointer", members=None)
  ens_head(INVALID, "null pointer", out3=None)
  ens_head(INVALID, "null pointer", ws=None)
  ens_head(INVALID, "bad head", head=3)
  ens_head(INVALID, "mixture type", mix=3)
  ens_head(UNSUPPORTED, "n_members", n=0)
  ens_head(UNSUPPORTED, "n_members", n=65)
  ens_head(INVALID, "dw must be NULL", mix=_lib.MIX_MATRIX, dw=P)
  ens_head(INVALID, "gammas missing", gammas=None)
  ens_head(INVALID, "is null", members=_lib.ptr_array([P, None]))
  ens_head(INVALID, "labels missing", labels=None)
  ens_head(INVALID, "labels missing", head=_lib.HEAD_MSE)
  ens_head(INVALID, "batch/dim", batch=0)
  ens_head(UNSUPPORTED, "dim 65", dim=65)
  ens_head(WORKSPACE, "workspace", ws_bytes=256)
  ens_head(UNSUPPORTED, "shared memory", n=64, dim=64)

  def head_loss(want, phrase, planes=False, **kw):
    a = dict(head=0, logits=P, labels=P, labels_f=None, loss_out=P, dlogits=None)
    a.update({k: kw.pop(k) for k in list(kw) if k in a})
    if planes:
      b = dict(planes=None, colsum=None, dz=0, batch=256, dim=10, ws=P, ws_bytes=BIG)
      b.update(kw)
      rejects("adn_head_loss_p", want, phrase, *a.values(), *b.values(), None)
    else:
      b = dict(batch=256, dim=10, ws=P, ws_bytes=BIG)
      b.update(kw)
      rejects("adn_head_loss", want, phrase, *a.values(), *b.values(), None)

  for planes in (False, True):
    head_loss(INVALID, "null pointer", planes, logits=None)
    head_loss(INVALID, "null pointer", planes, loss_out=None)
    head_loss(INVALID, "null pointer", planes, ws=None)
    head_loss(INVALID, "bad head", planes, head=5)
    head_loss(INVALID, "labels missing", planes, labels=None)
    head_loss(INVALID, "batch/dim", planes, batch=0)
    head_loss(UNSUPPORTED, "dim 65", planes, dim=65)
    head_loss(WORKSPACE, "workspace", planes, ws_bytes=256)
  head_loss(INVALID, "dz_log2_scale", True, dz=61)

  def fwd_p(want, phrase, **kw):
    a = dict(xp=P, wp=P, b=None, yp=P, y=None, batch=256, in_=64, out=32, act=0)
    a.update(kw)
    rejects("adn_dense_fwd_p", want, phrase, *a.values(), None)

  fwd_p(INVALID, "null pointer", xp=None)
  fwd_p(INVALID, "null pointer", wp=None)
  fwd_p(INVALID, "exactly one of yp / y", y=P)
  fwd_p(INVALID, "exactly one of yp / y", yp=None)
  fwd_p(INVALID, "bad shape", batch=0)
  fwd_p(INVALID, "bad shape", out=1 << 31)
  fwd_p(INVALID, "bad act", act=7)

  def bwd_p(want, phrase, **kw):
    a = dict(xp=P, wp=P, dzp=P, dxp=None, dx=None, dx_colsum=None, dw=P, batch=256, in_=64, out=32, mask=1, dz=0,
             ws=P, ws_bytes=BIG)
    a.update(kw)
    rejects("adn_dense_bwd_p", want, phrase, *a.values(), None)

  bwd_p(INVALID, "null pointer", xp=None)
  bwd_p(INVALID, "null pointer", dzp=None)
  bwd_p(INVALID, "null pointer", ws=None)
  bwd_p(INVALID, "wp required", wp=None, dxp=P)
  bwd_p(INVALID, "at most one of dxp / dx", dxp=P, dx=P)
  bwd_p(INVALID, "dx_colsum needs dx", dx_colsum=P)
  bwd_p(INVALID, "bad shape", in_=0)
  bwd_p(INVALID, "dz_log2_scale", dz=-61)

  # an output plane buffer off the alignment the TMA stores need, here at a 64 B offset
  fwd_p(INVALID, "yp: plane buffers must be 256 B aligned", yp=P + 64)
  bwd_p(INVALID, "dxp: plane buffers must be 256 B aligned", dxp=P + 64)
  fop = _lib.FwdOp(xp=P, wp=P, yp=P + 64, in_=64, out=32)
  rejects("adn_dense_fwd_p_group", INVALID, "yp: plane buffers must be 256 B aligned", ctypes.byref(fop), 1, 256, None)
  bop = _lib.BwdOp(xp=P, wp=P, dzp=P, dxp=P + 64, dw=P, in_=64, out=32, x_relu_mask=1, workspace=P, workspace_bytes=BIG)
  rejects("adn_dense_bwd_p_group", INVALID, "dxp: plane buffers must be 256 B aligned", ctypes.byref(bop), 1, 256, None)

  rejects("adn_colsum", INVALID, "null pointer", None, 256, 10, P, P, BIG, None)
  rejects("adn_colsum", INVALID, "null pointer", P, 256, 10, P, None, BIG, None)
  rejects("adn_colsum", INVALID, "bad shape", P, 0, 10, P, P, BIG, None)
  rejects("adn_colsum", WORKSPACE, "workspace", P, 256, 10, P, P, 64 * 10 * 4 - 1, None)

  def group(want, phrase, n=2, batch=256, dim=10, per_op=True, **kw):
    ops = (_lib.HeadOp * 2)()
    for o in ops:
      o.head, o.mixture_type, o.n_members, o.reg_multiplier = 0, 0, 2, 1.0
      o.members_host, o.gammas_host = ctypes.cast(members, ctypes.POINTER(ctypes.c_void_p)), gam
      o.w, o.labels, o.out3, o.workspace, o.workspace_bytes = P, P, P, P, BIG
    for k, v in kw.items():
      setattr(ops[1], k, v)
    rejects("adn_head_group", want, phrase, ops if n >= 0 else None, abs(n), batch, dim, None)
    if kw and per_op:
      assert "op 1" in lib.adn_last_error().decode()

  group(INVALID, "bad ops", n=-1)
  group(INVALID, "batch/dim", batch=0)
  group(INVALID, "batch/dim", dim=65)
  group(INVALID, "null pointer", workspace=None)
  group(INVALID, "null pointer", out3=None)
  group(INVALID, "bad head", head=3)
  group(INVALID, "mixture type", mixture_type=-1)
  group(UNSUPPORTED, "n_members", n_members=0)
  group(UNSUPPORTED, "n_members", n_members=65)
  group(INVALID, "dw must be NULL", mixture_type=_lib.MIX_MATRIX, dw=P)
  group(INVALID, "gammas missing", gammas_host=None)
  group(INVALID, "labels missing", labels=None)
  group(INVALID, "dz_log2_scale", dz_log2_scale=61)
  group(WORKSPACE, "workspace", workspace_bytes=256)
  group(UNSUPPORTED, "shared memory", dim=64, per_op=False, n_members=64)
  assert _lib.launch_count() == before


def test_engine_fails_loudly_without_gpu():
  import torch
  if torch.cuda.is_available():
    pytest.skip("GPU present")
  from adanet_b200 import _lib
  from adanet_b200.core import engine as eng
  with pytest.raises(_lib.AdnError):
    eng.IterationPlan(0, [], [], eng.EnsemblerPlanSpec(), 8, 4, 2)
