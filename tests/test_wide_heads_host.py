"""Host checks of the wide head kernel's entry point (adn_head_group_wide): argument validation before any launch,
the narrow / wide routing of ADN_Q_HEAD_PATH, and the conditioning of the wide-head parity configurations."""

import numpy as np
import pytest

from tests import parity_util as pu
from tests import wide_configs as wc

INVALID, UNSUPPORTED, WORKSPACE = -22, -95, -12
SENS_TOL = 5e-6


def test_wide_head_group_rejects_before_launch(built_lib):
  """Each malformed op is rejected with the right code and a message naming adn_head_group_wide and the op; the fake
  device pointers below are never dereferenced and nothing is launched."""
  from adanet_b200 import _lib
  P, BIG = 1 << 20, 1 << 40
  members = _lib.ptr_array([P + 256 * k for k in range(65)])
  gam = _lib.f32_array([0.5] * 65)
  before = _lib.launch_count()

  def op(**kw):
    a = dict(head=0, mixture_type=0, members_host=members, n_members=2, reg_is_zero=0, w=P, bias=None, gammas_host=gam,
             reg_multiplier=1.0, dz_log2_scale=0, labels=P, labels_f=None, out3=P, dw=None, dbias=None, dens=None,
             ens_out=None, dens_planes=None, colsum_only=0, reserved=0, workspace=P, workspace_bytes=BIG)
    a.update(kw)
    return _lib.HeadOp(**a)

  def rejects(want, phrase, ops, batch=256, dim=100):
    arr = (_lib.HeadOp * len(ops))(*ops)
    rc = built_lib.adn_head_group_wide(arr, len(ops), batch, dim, None)
    msg = built_lib.adn_last_error().decode()
    assert (rc, phrase in msg, "adn_head_group_wide" in msg) == (want, True, True), (phrase, rc, msg)
    return msg

  good = op()
  for bad, want, phrase in [
      (op(members_host=None), INVALID, "null pointer"),
      (op(out3=None), INVALID, "null pointer"),
      (op(workspace=None), INVALID, "null pointer"),
      (op(head=3), INVALID, "bad head"),
      (op(mixture_type=3), INVALID, "mixture type"),
      (op(n_members=0), UNSUPPORTED, "n_members"),
      (op(n_members=65), UNSUPPORTED, "n_members"),
      (op(mixture_type=_lib.MIX_MATRIX, dw=P), INVALID, "dw must be NULL"),
      (op(gammas_host=None), INVALID, "gammas missing"),
      (op(labels=None), INVALID, "labels missing"),
      (op(workspace_bytes=256), WORKSPACE, "workspace"),
  ]:
    # the bad op second: the message names it, and the good first op was not launched either
    msg = rejects(want, phrase, [good, bad])
    assert "op 1" in msg, msg
  rejects(UNSUPPORTED, "dim 0", [good], dim=0)
  rejects(UNSUPPORTED, "dim 16385", [good], dim=16385)
  rejects(INVALID, "bad batch", [good], batch=0)
  # the workspace the query gives is enough; one byte less is not
  need = _lib.query(_lib.Q_HEAD_WIDE_WS, 256, 100, 2)
  rejects(WORKSPACE, "workspace", [op(workspace_bytes=need - 257)])
  assert _lib.launch_count() == before


@pytest.mark.parametrize("dim,members,path", [(10, 44, 0), (10, 45, 1), (64, 6, 0), (64, 7, 1), (65, 1, 1),
                                              (1000, 64, 1), (1, 1, 0)])
def test_head_path_routing(built_lib, dim, members, path):
  """ADN_Q_HEAD_PATH: 0 exactly when the narrow kernel takes the op (dim <= 64 and its member slab fits shared
  memory), else 1; both workspace queries answer for any shape."""
  from adanet_b200 import _lib
  assert _lib.query(_lib.Q_HEAD_PATH, dim, members) == path
  assert _lib.query(_lib.Q_HEAD_WIDE_WS, 256, dim, members) > 0


def test_wide_workspace_covers_every_smaller_batch(built_lib):
  """A head sized for the static batch also runs on any prefix of it (ragged evaluation batches)."""
  from adanet_b200 import _lib
  for dim, members in ((100, 1), (100, 8), (1000, 64), (7, 3)):
    for batch in (48, 1000, 32768, 65537):
      have = _lib.query(_lib.Q_HEAD_WIDE_WS, batch, dim, members)
      for rows in sorted({1, 31, 32, 33, batch // 3, batch // 2 + 1, batch - 1, batch} - {0}):
        assert _lib.query(_lib.Q_HEAD_WIDE_WS, rows, dim, members) <= have, (dim, members, batch, rows)


def _max_trace_diff(a, b):
  worst = 0.0
  for ra, rb in zip(a, b):
    for name in ra.traces:
      for f in ("sub_loss", "ens_loss", "adanet_loss", "ema"):
        worst = max(worst, float(np.abs(np.asarray(ra.traces[name][f], np.float64) -
                                        np.asarray(rb.traces[name][f], np.float64)).max()))
  return worst


@pytest.mark.parametrize("name", sorted(wc.CONFIGS))
def test_wide_parity_configs_are_well_conditioned(name):
  """As test_parity_configs_are_well_conditioned: the oracle against itself with permuted input features and with
  2e-7 relative noise on every dense forward / weight gradient moves no per-step loss by 5e-6 or more."""
  cfg = wc.CONFIGS[name]
  d = cfg["data"][2]
  perm = np.random.default_rng(0).permutation(d)
  a, b = wc.oracle_run(cfg), wc.oracle_run(cfg, perm)
  assert [r.best_index for r in a] == [r.best_index for r in b]
  sens = _max_trace_diff(a, b)
  assert sens < SENS_TOL, "config %s is ill conditioned: oracle self-sensitivity %.3g" % (name, sens)
  for seed in (0, 1, 2):
    with pu.oracle_noise(2e-7, seed):
      c = wc.oracle_run(cfg)
    assert [r.best_index for r in a] == [r.best_index for r in c]
    sens = _max_trace_diff(a, c)
    assert sens < SENS_TOL, "config %s is ill conditioned: 2e-7 noise (seed %d) moves the oracle by %.3g" % (
        name, seed, sens)
