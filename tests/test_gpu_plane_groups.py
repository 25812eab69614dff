"""Grouped launches of the plane GEMM (csrc/planes.cu pl_gemm_kernel via adn_dense_fwd_p_group /
adn_dense_bwd_p_group), element by element against float64 NumPy, in both plane formats.

A group runs the tiles of up to MAX_GROUP = 8 problems per persistent launch; work items are numbered problem after
problem, a CTA carries its mbarrier ring from one problem into the next, and larger groups are split into several
launches.  Everything here checks what only groups exercise, plus epilogue branches that a group of one never takes:
the direct-epilogue dW un-scale, dx_mul (the dropout backward), dW-only ops without weights, and groups that mix
plane and dense outputs.

Bounds are componentwise: |err_ij| <= 3e-6 * (|A| |B|)_ij (+ 3e-6 |b_j| for a bias), where (|A| |B|) is the product
of the magnitudes.  A normwise bound against the largest entry cannot see a wrong small entry.  Operand entries are
drawn with magnitudes in [0.5, 2): in the fp16 format every operand then stays in fp16's normal range, where a plane
pair carries 22 significant bits (include/adanet_b200.h).
"""

import numpy as np
import pytest

from tests.test_gpu_planes import _layout, _merge, _planes

pytestmark = pytest.mark.gpu

TOL = 3e-6
ERR_WORKSPACE, ERR_UNSUPPORTED = -12, -95
DX_MUL = float(np.float32(1.0 / (1.0 - 0.25)))      # the dropout backward below a rate-0.25 layer

# forward ops: (in, out, bias, act, planes out, dropout (seed, layer) or None).  Ops with the same `in` read the same
# x planes, as the candidates of one iteration do.  Every op with out > 64 has a bias, so a bias missing from any
# column tile but the first shows in every such op.
FWD_G11 = [
    (1, 1, 1, 1, 1, None),
    (7, 3, 0, 0, 0, None),
    (64, 31, 1, 1, 1, (11, 0)),
    (64, 32, 1, 0, 0, None),
    (100, 33, 0, 1, 1, None),
    (257, 64, 1, 1, 1, (12, 1)),
    (1024, 65, 1, 0, 0, None),
    (4096, 200, 1, 1, 1, None),
    (100, 1024, 1, 1, 1, None),
    (7, 65, 1, 1, 0, None),
    (257, 200, 1, 0, 1, (13, 2)),
]
FWD_G17 = [
    (4096, 1, 1, 0, 0, None),
    (1, 1024, 1, 1, 1, None),
    (1024, 3, 0, 1, 1, (21, 0)),
    (257, 31, 1, 0, 0, None),
    (7, 200, 1, 1, 1, None),
    (100, 65, 1, 0, 1, None),
    (64, 1024, 1, 0, 0, None),
    (4096, 33, 1, 1, 1, (22, 1)),
    (257, 1, 0, 1, 1, None),
    (1, 64, 1, 0, 0, None),
    (64, 32, 1, 1, 1, (23, 2)),
    (100, 3, 1, 1, 0, None),
    (7, 31, 0, 0, 1, None),
    (1024, 200, 1, 1, 1, None),
    (4096, 65, 1, 1, 0, None),
    (257, 1024, 1, 1, 1, None),
    (64, 64, 0, 1, 1, (24, 3)),
]
# batch 128: one-tile problems between problems of 266, 141 and 79 tiles, so the 132 CTAs of a launch cross problem
# boundaries (and K) several times each
FWD_WRAP = [
    (64, 1, 1, 1, 1, None),
    (100, 17000, 1, 1, 1, None),
    (7, 3, 0, 0, 0, None),
    (257, 9000, 1, 0, 0, None),
    (1024, 64, 1, 1, 1, (31, 0)),
    (4096, 33, 1, 0, 1, None),
    (1, 5000, 1, 1, 1, None),
    (64, 31, 1, 0, 0, None),
    (100, 300, 1, 1, 1, None),
]
FWD_CASES = ([("g11", FWD_G11, b) for b in (1, 37, 128, 129, 1000, 4097)] +
             [("g17", FWD_G17, b) for b in (37, 129, 4097)] + [("wrap", FWD_WRAP, 128)])
DROP_RATE = 0.25
DROP_STEP = 3

# backward ops: (in, out, x_relu_mask, dz_log2_scale, dx_mul (0 = 1), outputs).  "dw" only: no weights (wp = NULL),
# how MATRIX mixture weights run.  The dW split-K caps (max_dw_splits: 16M floats of partials) are 64 for every op
# but 520 x 520 (62).
BWD_OPS = [
    (64, 32, 1, 0, 0.0, "dw dxp cs"),
    (100, 10, 0, 7, 0.0, "dw"),
    (257, 65, 1, 15, DX_MUL, "dx cs"),
    (33, 129, 0, 7, DX_MUL, "dw dxp cs"),
    (520, 520, 1, 15, 0.0, "dw"),
    (7, 3, 1, 0, DX_MUL, "dw dxp"),
    (200, 1, 0, 15, 0.0, "dw dx"),
    (1, 64, 1, 7, 0.0, "dw"),
    (129, 200, 0, 0, DX_MUL, "dxp cs"),
    (1024, 64, 0, 7, 0.0, "dw dx cs"),
]


def _open():
  import torch
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  lib = _lib.load()
  _lib.check(lib.adn_init(), "adn_init")
  return torch, _lib, lib


def _set_format(_lib, name):
  _lib.set_plane_format(_lib.PLANES_F16 if name == "f16" else _lib.PLANES_TF32)


@pytest.fixture(scope="module", params=["f16", "tf32"])
def env(request):
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _set_format(_lib, request.param)
  _lib.plane_overflow()      # clear the sticky flag
  yield torch, _lib, lib
  _lib.set_plane_format(before)


def _stream(torch):
  return torch.cuda.current_stream().cuda_stream


def _mag(rng, shape):
  """random signs, magnitudes uniform in [0.5, 2)"""
  return (rng.uniform(0.5, 2.0, shape) * rng.choice([-1.0, 1.0], shape)).astype(np.float32)


def _bits_of(pos):
  """[r, nb32 * 32] bool -> sign-bit words [nb32, r]"""
  r = pos.shape[0]
  return (pos.reshape(r, -1, 32) * (np.uint64(1) << np.arange(32, dtype=np.uint64))).sum(axis=2).astype(np.uint32).T


def _cw(got, exact, bound, what):
  """[] if |got - exact| <= bound everywhere, else one line describing the worst entry"""
  err = np.abs(got.astype(np.float64) - exact)
  bad = ~(err <= bound)
  if not bad.any():
    return []
  ratio = np.where(np.isnan(err) | (bound <= 0), np.inf, err / np.maximum(bound, 1e-300))
  i = np.unravel_index(int(np.nanargmax(np.where(bad, ratio, -1.0))), got.shape)
  return ["%s: %d of %d entries beyond the componentwise bound, worst err/bound %.3g at %s (got %r, want %r)" %
          (what, int(bad.sum()), bad.size, float(ratio[i]), i, float(got[i]), float(exact[i]))]


def _bytes_equal(a, b):
  import torch
  return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------------------------
def _fwd_case(torch, _lib, lib, B, spec, seed):
  """host data + operand planes of every op of a forward group"""
  rng = np.random.default_rng(seed)
  xs = {i: _mag(rng, (B, i)) for i in sorted({s[0] for s in spec})}
  xps = {i: _planes(torch, _lib, lib, a) for i, a in xs.items()}
  ops = []
  for I, O, has_b, act, planes, drop in spec:
    w = (_mag(rng, (I, O)) / np.sqrt(I)).astype(np.float32)
    b = _mag(rng, (O,)) if has_b else None
    ops.append(dict(I=I, O=O, act=act, planes=planes, drop=drop, x=xs[I], w=w, b=b, xp=xps[I],
                    wp=_planes(torch, _lib, lib, w), bd=torch.as_tensor(b).cuda() if has_b else None))
  step_dev = torch.full((), DROP_STEP, dtype=torch.int64, device="cuda")
  return dict(B=B, ops=ops, step_dev=step_dev)


def _fwd_buf(torch, _lib, B, d):
  if d["planes"]:
    return torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, d["O"]) // 4,), device="cuda")
  return torch.full((B, d["O"]), float("nan"), device="cuda")


def _fwd_struct(_lib, case, d, buf):
  op = _lib.FwdOp(d["xp"].data_ptr(), d["wp"].data_ptr(), d["bd"].data_ptr() if d["bd"] is not None else None,
                  buf.data_ptr() if d["planes"] else None, None if d["planes"] else buf.data_ptr(), d["I"], d["O"],
                  d["act"], 0)
  if d["drop"]:
    op.dropout_rate, op.dropout_seed, op.dropout_layer = DROP_RATE, d["drop"][0], d["drop"][1]
    op.dropout_step_dev = case["step_dev"].data_ptr()
  return op


def _fwd_run(torch, _lib, lib, case, idx):
  """runs ops[idx] as one group call into fresh output buffers; returns the buffers"""
  B = case["B"]
  bufs = [_fwd_buf(torch, _lib, B, case["ops"][i]) for i in idx]
  structs = [_fwd_struct(_lib, case, case["ops"][i], buf) for i, buf in zip(idx, bufs)]
  _lib.check(lib.adn_dense_fwd_p_group((_lib.FwdOp * len(structs))(*structs), len(structs), B, _stream(torch)),
             "adn_dense_fwd_p_group")
  return bufs


def _fwd_check(torch, _lib, lib, case, k, buf):
  """failures (list of strings) of op k against float64"""
  from tests.parity_util import orc
  d, B = case["ops"][k], case["B"]
  x64, w64 = d["x"].astype(np.float64), d["w"].astype(np.float64)
  exact = x64 @ w64
  bound = TOL * (np.abs(x64) @ np.abs(w64))
  if d["b"] is not None:
    exact += d["b"]
    bound += TOL * np.abs(d["b"].astype(np.float64))
  if d["act"]:
    exact = np.maximum(exact, 0.0)
  what = "op %d (in %d, out %d%s)" % (k, d["I"], d["O"], ", dropout" if d["drop"] else "")
  fails = []
  if d["drop"]:
    keep = orc.dropout_keep_mask(d["drop"][0], d["drop"][1], DROP_STEP, B, d["O"], DROP_RATE)
    pre = exact
    exact = np.where(keep, pre / (1.0 - DROP_RATE), 0.0)
    bound = bound / (1.0 - DROP_RATE)
  got = _merge(torch, _lib, lib, buf, B, d["O"]) if d["planes"] else buf.cpu().numpy()
  fails += _cw(got, exact, bound, what)
  if d["drop"]:
    if not (got[~keep] == 0).all():
      fails.append("%s: a dropped entry is nonzero" % what)
    clear = np.abs(pre) > 2 * bound          # the value is nonzero whatever the rounding: zero iff dropped
    if not np.array_equal(got[clear] != 0, keep[clear]):
      fails.append("%s: the dropout mask differs from orc.dropout_keep_mask" % what)
  if d["planes"]:
    hi, bits, bk = _layout(_lib, buf, B, d["O"])
    if d["O"] % bk and not (hi[-1, :, d["O"] % bk:] == 0).all():
      fails.append("%s: K padding of the output planes is not zero" % what)
    # (against the stored value, not the hi plane alone: an fp32 result in (0, 2^-25] has hi = +0 and lo' > 0)
    pos = np.zeros((B, bits.shape[0] * 32), dtype=bool)
    pos[:, :d["O"]] = got > 0
    if not np.array_equal(bits, _bits_of(pos)):
      fails.append("%s: sign bits disagree with the stored values" % what)
  return fails


@pytest.mark.parametrize("name,spec,B", FWD_CASES, ids=["%s-b%d" % (n, b) for n, _, b in FWD_CASES])
def test_fwd_group(env, name, spec, B):
  """Every op of a heterogeneous group (2-3 launches) within the componentwise bound, and byte for byte what the
  same op computes launched alone: a tile is computed by one CTA in a fixed order whatever the grouping."""
  torch, _lib, lib = env
  case = _fwd_case(torch, _lib, lib, B, spec, seed=B * 31 + len(spec))
  n = len(spec)
  group = _fwd_run(torch, _lib, lib, case, list(range(n)))
  fails = []
  for k in range(n):
    fails += _fwd_check(torch, _lib, lib, case, k, group[k])
    alone = _fwd_run(torch, _lib, lib, case, [k])[0]
    if not _bytes_equal(group[k], alone):
      fails.append("op %d: grouped output differs from the op launched alone" % k)
  assert not fails, "\n".join(fails)


# ------------------------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------------------------
def _bwd_case(torch, _lib, lib, B, spec, seed):
  rng = np.random.default_rng(seed)
  ops = []
  for I, O, mask, s, mul, outs in spec:
    outs = set(outs.split())
    x = _mag(rng, (B, I))
    if mask:
      x = np.maximum(x, 0)          # a ReLU output: the mask is x > 0
    dz = (_mag(rng, (B, O)) * 2.0 ** -s).astype(np.float32)     # the planes carry dz * 2^s = O(1)
    needs_w = bool(outs & {"dxp", "dx"})
    w = (_mag(rng, (I, O)) / np.sqrt(O)).astype(np.float32) if needs_w else None
    ops.append(dict(I=I, O=O, mask=mask, s=s, mul=mul, outs=outs, x=x, dz=dz, w=w,
                    xp=_planes(torch, _lib, lib, x), dzp=_planes(torch, _lib, lib, dz, s),
                    wp=_planes(torch, _lib, lib, w) if needs_w else None,
                    ws_bytes=_lib.query(_lib.Q_DENSE_BWD_P_WS, B, I, O)))
  return dict(B=B, ops=ops)


def _bwd_bufs(torch, _lib, B, d):
  I, O = d["I"], d["O"]
  f = dict(dw=None, dxp=None, dx=None, cs=None)
  if "dw" in d["outs"]:
    f["dw"] = torch.full((I, O), float("nan"), device="cuda")
  if "dxp" in d["outs"]:
    f["dxp"] = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, I) // 4,), device="cuda")
  if "dx" in d["outs"]:
    f["dx"] = torch.full((B, I), float("nan"), device="cuda")
  if "cs" in d["outs"]:
    f["cs"] = torch.full((I,), float("nan"), device="cuda")
  f["ws"] = torch.empty((d["ws_bytes"],), dtype=torch.uint8, device="cuda")
  return f


def _bwd_struct(_lib, d, f, ws_bytes=None):
  ptr = lambda t: t.data_ptr() if t is not None else None
  return _lib.BwdOp(d["xp"].data_ptr(), ptr(d["wp"]), d["dzp"].data_ptr(), ptr(f["dxp"]), ptr(f["dx"]), ptr(f["cs"]),
                    ptr(f["dw"]), d["I"], d["O"], d["mask"], d["s"], f["ws"].data_ptr(),
                    d["ws_bytes"] if ws_bytes is None else ws_bytes, d["mul"], 0.0)


def _bwd_call(torch, _lib, lib, B, structs):
  return lib.adn_dense_bwd_p_group((_lib.BwdOp * len(structs))(*structs), len(structs), B, _stream(torch))


def _bwd_run(torch, _lib, lib, case, idx):
  B = case["B"]
  bufs = [_bwd_bufs(torch, _lib, B, case["ops"][i]) for i in idx]
  structs = [_bwd_struct(_lib, case["ops"][i], f) for i, f in zip(idx, bufs)]
  _lib.check(_bwd_call(torch, _lib, lib, B, structs), "adn_dense_bwd_p_group")
  return bufs


def _bwd_exact(d, x=None):
  """float64 (dw, dw bound, dx, dx bound) of one op; dx un-scaled (the true gradient times dx_mul)"""
  x64 = (d["x"] if x is None else x).astype(np.float64)
  dz64 = d["dz"].astype(np.float64)
  dw = x64.T @ dz64
  dw_b = TOL * (np.abs(x64).T @ np.abs(dz64))
  dx = dx_b = None
  if d["w"] is not None:
    w64 = d["w"].astype(np.float64)
    m = (x64 > 0) if d["mask"] else 1.0
    mul = d["mul"] or 1.0
    dx = (dz64 @ w64.T) * m * mul
    dx_b = TOL * (np.abs(dz64) @ np.abs(w64).T) * m * mul
  return dw, dw_b, dx, dx_b


def _bwd_check(torch, _lib, lib, case, k, f, x=None):
  d, B = case["ops"][k], case["B"]
  what = "op %d (in %d, out %d, mask %d, scale 2^%d, dx_mul %g)" % (k, d["I"], d["O"], d["mask"], d["s"], d["mul"] or 1)
  dw, dw_b, dx, dx_b = _bwd_exact(d, x)
  fails = []
  if f["dw"] is not None:
    fails += _cw(f["dw"].cpu().numpy(), dw, dw_b, what + " dw")
  if f["dxp"] is not None:          # the planes keep the gradient's scale
    fails += _cw(_merge(torch, _lib, lib, f["dxp"], B, d["I"]) / 2.0 ** d["s"], dx, dx_b, what + " dxp")
  if f["dx"] is not None:           # dense fp32 comes back un-scaled
    fails += _cw(f["dx"].cpu().numpy(), dx, dx_b, what + " dx")
  if f["cs"] is not None:
    fails += _cw(f["cs"].cpu().numpy(), dx.sum(axis=0), dx_b.sum(axis=0) + TOL * np.abs(dx).sum(axis=0), what + " colsum")
  return fails


@pytest.mark.parametrize("B", [37, 256, 8192, 32768])
def test_bwd_group(env, B):
  """A 10-op backward group: dW with and without dX, dX as planes and dense, with and without the ReLU mask, column
  sums, gradient scales 2^0 / 2^7 / 2^15 and dx_mul.  At batch 37 and 256 dW takes the direct epilogue (one split,
  un-scaled there); at 8192 and 32768 it is split over K and un-scaled by the reduction.  dX is byte-identical to
  the op launched alone; a repeated group call (memoized split size) is byte-identical in every output.  dW alone may
  legitimately differ from the group: the split size is chosen for the whole group."""
  torch, _lib, lib = env
  case = _bwd_case(torch, _lib, lib, B, BWD_OPS, seed=B + 17)
  n = len(BWD_OPS)
  first = _bwd_run(torch, _lib, lib, case, list(range(n)))
  fails = []
  for k in range(n):
    fails += _bwd_check(torch, _lib, lib, case, k, first[k])
  again = _bwd_run(torch, _lib, lib, case, list(range(n)))
  for k in range(n):
    for key in ("dw", "dxp", "dx", "cs"):
      if first[k][key] is not None and not _bytes_equal(first[k][key], again[k][key]):
        fails.append("op %d: %s differs between two identical group calls" % (k, key))
    alone = _bwd_run(torch, _lib, lib, case, [k])[0]
    for key in ("dxp", "dx"):
      if first[k][key] is not None and not _bytes_equal(first[k][key], alone[key]):
        fails.append("op %d: grouped %s differs from the op launched alone" % (k, key))
  assert not _lib.plane_overflow()
  assert not fails, "\n".join(fails)


def test_bwd_group_split_cap(env):
  """dW of one 2048 x 1024 layer beside fifteen 1 x 1 ones at batch 32768.  The planner in dense_bwd_group picks a
  split size for the whole group (40 k-blocks per work item with fp16 planes, 79 with TF32) that would need more
  partial sums than the large layer's workspace holds (max_dw_splits: 8), so that layer alone runs with a larger
  split size (64 / 128 k-blocks) while the small ones keep the group's."""
  torch, _lib, lib = env
  B = 32768
  spec = [(2048, 1024, 0, 15, 0.0, "dw")] + [(1, 1, k % 2, (0, 7, 15)[k % 3], 0.0, "dw") for k in range(15)]
  case = _bwd_case(torch, _lib, lib, B, spec, seed=5)
  bufs = _bwd_run(torch, _lib, lib, case, list(range(len(spec))))
  fails = []
  for k in range(len(spec)):
    fails += _bwd_check(torch, _lib, lib, case, k, bufs[k])
  assert not fails, "\n".join(fails)


def test_fwd_dropout_then_bwd_group(env):
  """Three candidates' dropout forward (one group) feeding their backward (one group) with dx_mul = 1/(1-rate): dX is
  (dz w^T) * keep * (relu > 0) / (1-rate), the mask read from the sign bits the forward wrote.  The third runs rows
  1000..1999 of a minibatch (dropout_row0 = 1000, a row-sharded candidate): its mask is those rows of the whole
  minibatch's mask, not the first 1000 rows'."""
  torch, _lib, lib = env
  from tests.parity_util import orc
  B, I, H, O, s = 1000, 100, 257, 65, 7
  rng = np.random.default_rng(41)
  step_dev = torch.full((), DROP_STEP, dtype=torch.int64, device="cuda")
  cands = []
  for c, (seed, layer, row0) in enumerate(((51, 1, 0), (52, 2, 0), (51, 1, 1000))):
    x = _mag(rng, (B, I))
    w1 = (_mag(rng, (I, H)) / np.sqrt(I)).astype(np.float32)
    b1 = _mag(rng, (H,))
    w2 = (_mag(rng, (H, O)) / np.sqrt(O)).astype(np.float32)
    dz = (_mag(rng, (B, O)) * 2.0 ** -s).astype(np.float32)
    cands.append(dict(seed=seed, layer=layer, row0=row0, x=x, w1=w1, b1=b1, w2=w2, dz=dz, xp=_planes(torch, _lib, lib, x),
                      w1p=_planes(torch, _lib, lib, w1), b1d=torch.as_tensor(b1).cuda(), w2p=_planes(torch, _lib, lib, w2),
                      dzp=_planes(torch, _lib, lib, dz, s),
                      hp=torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, H) // 4,), device="cuda")))
  fops = []
  for c in cands:
    op = _lib.FwdOp(c["xp"].data_ptr(), c["w1p"].data_ptr(), c["b1d"].data_ptr(), c["hp"].data_ptr(), None, I, H, 1, 0)
    op.dropout_rate, op.dropout_seed, op.dropout_layer = DROP_RATE, c["seed"], c["layer"]
    op.dropout_row0, op.dropout_step_dev = c["row0"], step_dev.data_ptr()
    fops.append(op)
  _lib.check(lib.adn_dense_fwd_p_group((_lib.FwdOp * 3)(*fops), 3, B, _stream(torch)), "adn_dense_fwd_p_group")
  bops, bufs = [], []
  for c in cands:
    d = dict(I=H, O=O, mask=1, s=s, mul=DX_MUL, outs={"dw", "dxp", "cs"}, x=None, dz=c["dz"], w=c["w2"], xp=c["hp"],
             dzp=c["dzp"], wp=c["w2p"], ws_bytes=_lib.query(_lib.Q_DENSE_BWD_P_WS, B, H, O))
    bops.append(d)
    bufs.append(_bwd_bufs(torch, _lib, B, d))
  _lib.check(_bwd_call(torch, _lib, lib, B, [_bwd_struct(_lib, d, f) for d, f in zip(bops, bufs)]),
             "adn_dense_bwd_p_group")
  fails = []
  for k, c in enumerate(cands):
    h = _merge(torch, _lib, lib, c["hp"], B, H)          # the activation the backward read
    _, bits, _ = _layout(_lib, c["hp"], B, H)
    nb32 = bits.shape[0]
    pos = np.zeros((B, nb32 * 32), dtype=bool)
    pos[:, :H] = h > 0
    assert np.array_equal(bits, _bits_of(pos))
    keep = orc.dropout_keep_mask(c["seed"], c["layer"], DROP_STEP, c["row0"] + B, H, DROP_RATE)[c["row0"]:]
    x64, w164 = c["x"].astype(np.float64), c["w1"].astype(np.float64)
    relu = np.maximum(x64 @ w164 + c["b1"], 0.0)
    assert not (pos[:, :H] & ~keep).any()
    clear = relu > 2 * TOL * (np.abs(x64) @ np.abs(w164) + np.abs(c["b1"].astype(np.float64)))
    assert np.array_equal(pos[:, :H][clear], keep[clear])
    mask = keep & (h > 0)
    dz64, w64 = c["dz"].astype(np.float64), c["w2"].astype(np.float64)
    want = (dz64 @ w64.T) * mask / (1.0 - DROP_RATE)
    bound = TOL * (np.abs(dz64) @ np.abs(w64).T) * mask / (1.0 - DROP_RATE)
    fails += _cw(_merge(torch, _lib, lib, bufs[k]["dxp"], B, H) / 2.0 ** s, want, bound, "cand %d dxp" % k)
    fails += _cw(bufs[k]["cs"].cpu().numpy(), want.sum(axis=0), bound.sum(axis=0) + TOL * np.abs(want).sum(axis=0),
                 "cand %d colsum" % k)
    h64 = h.astype(np.float64)
    fails += _cw(bufs[k]["dw"].cpu().numpy(), h64.T @ dz64, TOL * (np.abs(h64).T @ np.abs(dz64)), "cand %d dw" % k)
  assert not fails, "\n".join(fails)


def test_bwd_group_errors(env):
  """One op a byte short of workspace: ADN_ERR_WORKSPACE naming that op, and no output of any op is written.
  n = 0 is a no-op; n = 257 is refused."""
  torch, _lib, lib = env
  B = 256
  case = _bwd_case(torch, _lib, lib, B, BWD_OPS[:4], seed=99)
  bufs = [_bwd_bufs(torch, _lib, B, d) for d in case["ops"]]
  for f in bufs:
    if f["dxp"] is not None:
      f["dxp"].fill_(float("nan"))
  structs = [_bwd_struct(_lib, d, f, d["ws_bytes"] - (k == 2)) for k, (d, f) in enumerate(zip(case["ops"], bufs))]
  assert _bwd_call(torch, _lib, lib, B, structs) == ERR_WORKSPACE
  assert "op 2 " in lib.adn_last_error().decode()
  torch.cuda.synchronize()
  for k, f in enumerate(bufs):
    for key in ("dw", "dxp", "dx", "cs"):
      if f[key] is not None:
        assert torch.isnan(f[key]).all(), "op %d: %s written by a failed group call" % (k, key)
  sp = _stream(torch)
  assert lib.adn_dense_bwd_p_group(None, 0, B, sp) == 0
  assert lib.adn_dense_fwd_p_group(None, 0, B, sp) == 0
  assert lib.adn_dense_bwd_p_group((_lib.BwdOp * 257)(), 257, B, sp) == ERR_UNSUPPORTED
  assert lib.adn_dense_fwd_p_group((_lib.FwdOp * 257)(), 257, B, sp) == ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------------------------------
# non-cancelling operands and wide dynamic range
# ------------------------------------------------------------------------------------------------------------------
# (the inputs are functions so that tests/probe_accuracy.py measures the same ones)
def positive_fwd_inputs():
  """x [512, 4096], w [4096, 256], all entries positive"""
  rng = np.random.default_rng(61)
  x = np.abs(_mag(rng, (512, 4096)))
  w = (np.abs(_mag(rng, (4096, 256))) / np.sqrt(4096)).astype(np.float32)
  return x, w


def positive_dw_inputs():
  """x [32768, 100] = relu(.) >= 0, dz [32768, 192] > 0 of magnitude 2^-15, and the log2 scale of its planes"""
  s = 15
  rng = np.random.default_rng(62)
  x = np.maximum(_mag(rng, (32768, 100)), 0)
  dz = (np.abs(_mag(rng, (32768, 192))) * 2.0 ** -s).astype(np.float32)
  return x, dz, s


def row_spread_inputs():
  """x [1000, 1024] and dz [1000, 200] with rows scaled by 2^e, e in [-8, 8]; w [1024, 200]"""
  rng = np.random.default_rng(63)
  x = (_mag(rng, (1000, 1024)) * np.exp2(rng.integers(-8, 9, 1000))[:, None]).astype(np.float32)
  w = (_mag(rng, (1024, 200)) / np.sqrt(1024)).astype(np.float32)
  dz = (_mag(rng, (1000, 200)) * np.exp2(rng.integers(-8, 9, 1000))[:, None]).astype(np.float32)
  return x, w, dz


def test_all_positive_fwd(env):
  """x, w > 0 at K = 4096: no cancellation, so the truncating accumulation inside the tensor core adds up instead
  of averaging out.  The 128-K chunks re-accumulated with round-to-nearest keep every entry within 3e-6 of itself."""
  torch, _lib, lib = env
  x, w = positive_fwd_inputs()
  (B, I), O = x.shape, w.shape[1]
  exact = x.astype(np.float64) @ w.astype(np.float64)
  xp, wp = _planes(torch, _lib, lib, x), _planes(torch, _lib, lib, w)
  sp = _stream(torch)
  y = torch.full((B, O), float("nan"), device="cuda")
  yp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, O) // 4,), device="cuda")
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, None, y.data_ptr(), B, I, O, 0, sp), "fwd_p")
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, yp.data_ptr(), None, B, I, O, 0, sp), "fwd_p")
  fails = _cw(y.cpu().numpy(), exact, TOL * exact, "dense") + \
      _cw(_merge(torch, _lib, lib, yp, B, O), exact, TOL * exact, "planes")
  assert not fails, "\n".join(fails)


def test_all_positive_dw_split_k(env):
  """dW = x^T dz with x = relu(.) >= 0, dz > 0, K = batch = 32768 at dz scale 2^15: the split-K partials and their
  fixed-order reduction keep every entry within 3e-6 of itself."""
  torch, _lib, lib = env
  x, dz, s = positive_dw_inputs()
  (B, I), O = x.shape, dz.shape[1]
  exact = x.astype(np.float64).T @ dz.astype(np.float64)
  xp, dzp = _planes(torch, _lib, lib, x), _planes(torch, _lib, lib, dz, s)
  nb = _lib.query(_lib.Q_DENSE_BWD_P_WS, B, I, O)
  ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")
  dw = torch.full((I, O), float("nan"), device="cuda")
  _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), None, dzp.data_ptr(), None, None, None, dw.data_ptr(), B, I, O, 1, s,
                                 ws.data_ptr(), nb, _stream(torch)), "bwd_p")
  fails = _cw(dw.cpu().numpy(), exact, TOL * exact, "dw")
  assert not fails, "\n".join(fails)


def test_row_magnitudes(env):
  """Rows of x (forward) and of dz (dX) scaled by 2^e, e in [-8, 8], and dW over those rows: each row is held to
  the bound of its own magnitude."""
  torch, _lib, lib = env
  x, w, dz = row_spread_inputs()
  (B, I), O = x.shape, w.shape[1]
  x64, w64 = x.astype(np.float64), w.astype(np.float64)
  sp = _stream(torch)
  xp, wp = _planes(torch, _lib, lib, x), _planes(torch, _lib, lib, w)
  y = torch.full((B, O), float("nan"), device="cuda")
  _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, None, y.data_ptr(), B, I, O, 0, sp), "fwd_p")
  fails = _cw(y.cpu().numpy(), x64 @ w64, TOL * (np.abs(x64) @ np.abs(w64)), "fwd")
  # backward of the same layer: dz rows spread the same way
  dz64 = dz.astype(np.float64)
  dzp = _planes(torch, _lib, lib, dz)
  nb = _lib.query(_lib.Q_DENSE_BWD_P_WS, B, I, O)
  ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")
  dw = torch.full((I, O), float("nan"), device="cuda")
  dx = torch.full((B, I), float("nan"), device="cuda")
  _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), wp.data_ptr(), dzp.data_ptr(), None, dx.data_ptr(), None,
                                 dw.data_ptr(), B, I, O, 0, 0, ws.data_ptr(), nb, sp), "bwd_p")
  fails += _cw(dx.cpu().numpy(), dz64 @ w64.T, TOL * (np.abs(dz64) @ np.abs(w64).T), "dx")
  fails += _cw(dw.cpu().numpy(), x64.T @ dz64, TOL * (np.abs(x64).T @ np.abs(dz64)), "dw")
  assert not fails, "\n".join(fails)


def test_tf32_power_of_two_rows_commute(env):
  """TF32 planes have fp32's exponent range and no subnormals here, so every rounding of the pipeline commutes with
  a power of two: Y(diag(2^e) X) is diag(2^e) Y(X) bit for bit, in dense and plane outputs, and likewise dX.  (Not
  so for fp16 planes: a lo' in fp16's subnormal range legitimately breaks it.)"""
  torch, _lib, lib = env
  if _lib.plane_format() != _lib.PLANES_TF32:
    pytest.skip("exact only in the TF32 format")
  B, I, O = 1000, 1024, 200
  rng = np.random.default_rng(64)
  e = np.exp2(rng.integers(-8, 9, B)).astype(np.float32)[:, None]
  x = _mag(rng, (B, I))
  w = (_mag(rng, (I, O)) / np.sqrt(I)).astype(np.float32)
  dz = _mag(rng, (B, O))
  wp = _planes(torch, _lib, lib, w)
  sp = _stream(torch)
  nb = _lib.query(_lib.Q_DENSE_BWD_P_WS, B, I, O)
  ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")
  res = []
  for xs, dzs in ((x, dz), (x * e, dz * e)):
    xp, dzp = _planes(torch, _lib, lib, xs), _planes(torch, _lib, lib, dzs)
    y = torch.empty((B, O), device="cuda")
    yp = torch.zeros((_lib.query(_lib.Q_PLANES_BYTES, B, O) // 4,), device="cuda")
    dx = torch.empty((B, I), device="cuda")
    _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, None, y.data_ptr(), B, I, O, 1, sp), "fwd_p")
    _lib.check(lib.adn_dense_fwd_p(xp.data_ptr(), wp.data_ptr(), None, yp.data_ptr(), None, B, I, O, 1, sp), "fwd_p")
    _lib.check(lib.adn_dense_bwd_p(xp.data_ptr(), wp.data_ptr(), dzp.data_ptr(), None, dx.data_ptr(), None, None, B, I,
                                   O, 0, 0, ws.data_ptr(), nb, sp), "bwd_p")
    res.append((y.cpu().numpy(), _merge(torch, _lib, lib, yp, B, O), dx.cpu().numpy()))
  for a, b in zip(*res):
    assert np.array_equal(a * e, b)

