"""Multi-source forward ops of the grouped plane GEMM (adn_fwd_op.srcs / n_srcs, csrc/planes.cu pl_gemm_ms_kernel),
element by element against float64 NumPy, in both plane formats.

A multi-source op computes y = act(x_0 w_0 + x_1 w_1 + ... + b): a dense layer over concat([x_0, x_1, ...], axis=-1)
whose kernel is split into row blocks, each piece its own plane tensor.  That is how an AdaNet subnetwork reads the
hidden layers of the subnetworks already in the ensemble.  The float64 reference is the single-matrix product over
the materialised concatenation, with the componentwise bound of tests/test_gpu_plane_groups.py.

Piece widths are chosen off and on the k-block grid of both formats (32 and 64 columns), with up to
ADN_FWD_MAX_SRCS = 3 extra pieces; the epilogues are ReLU and linear, planes and dense out, with and without dropout.
"""

import ctypes

import numpy as np
import pytest

from tests.test_gpu_plane_groups import (_bytes_equal, _fwd_buf, _fwd_check, _fwd_struct, _mag, _planes, _stream,
                                         env)  # noqa: F401  (env: the per-format fixture)

pytestmark = pytest.mark.gpu

ERR_INVALID = -22

# multi-source ops: (piece widths [own, extra...], out, bias, act, planes out, dropout (seed, layer) or None)
MS_OPS = [
    ([100, 37], 65, 1, 1, 1, None),
    ([64, 64], 64, 1, 0, 0, None),
    ([1, 129], 200, 1, 1, 1, (41, 0)),
    ([37, 64, 200], 33, 0, 1, 1, None),
    ([3, 300, 1, 65], 129, 1, 1, 1, (42, 1)),
    ([257, 100], 1, 1, 0, 0, None),
    ([32, 32, 32, 32], 31, 1, 0, 1, None),
    ([129, 1], 1024, 1, 1, 0, None),
]
# single-source ops that share a group with them
SS_OPS = [
    ([64], 32, 1, 1, 1, None),
    ([100], 65, 0, 0, 0, None),
    ([257], 200, 1, 1, 1, (43, 2)),
]


def _case(torch, _lib, lib, B, spec, seed):
  """host data and planes: every piece its own x and w plane tensor; d["x"] / d["w"] are the concatenations"""
  rng = np.random.default_rng(seed)
  ops = []
  for widths, O, has_b, act, planes, drop in spec:
    K = sum(widths)
    xs = [_mag(rng, (B, i)) for i in widths]
    ws = [(_mag(rng, (i, O)) / np.sqrt(K)).astype(np.float32) for i in widths]
    b = _mag(rng, (O,)) if has_b else None
    ops.append(dict(I=K, O=O, act=act, planes=planes, drop=drop, widths=widths, b=b,
                    x=np.concatenate(xs, axis=1), w=np.concatenate(ws, axis=0),
                    xps=[_planes(torch, _lib, lib, a) for a in xs], wps=[_planes(torch, _lib, lib, a) for a in ws],
                    bd=torch.as_tensor(b).cuda() if has_b else None))
  step_dev = torch.full((), 3, dtype=torch.int64, device="cuda")
  return dict(B=B, ops=ops, step_dev=step_dev)


def _struct(_lib, case, d, buf, keep):
  """adn_fwd_op of d: piece 0 in xp / wp, the others in srcs (the ctypes array is appended to `keep`)"""
  d = dict(d, xp=d["xps"][0], wp=d["wps"][0], I=d["widths"][0])
  op = _fwd_struct(_lib, case, d, buf)
  extra = len(d["widths"]) - 1
  if extra:
    arr = (_lib.FwdSrc * extra)(*[_lib.FwdSrc(x.data_ptr(), w.data_ptr(), i)
                                  for x, w, i in zip(d["xps"][1:], d["wps"][1:], d["widths"][1:])])
    keep.append(arr)
    op.srcs = ctypes.cast(arr, ctypes.POINTER(_lib.FwdSrc))
    op.n_srcs = extra
  return op


def _call(torch, _lib, lib, B, structs):
  return lib.adn_dense_fwd_p_group((_lib.FwdOp * len(structs))(*structs), len(structs), B, _stream(torch))


def _run(torch, _lib, lib, case, idx):
  B, keep = case["B"], []
  bufs = [_fwd_buf(torch, _lib, B, case["ops"][i]) for i in idx]
  structs = [_struct(_lib, case, case["ops"][i], buf, keep) for i, buf in zip(idx, bufs)]
  _lib.check(_call(torch, _lib, lib, B, structs), "adn_dense_fwd_p_group")
  return bufs


@pytest.mark.parametrize("B", [1, 37, 129, 1000])
def test_multi_source_group(env, B):
  """Every op of a group that mixes multi-source and single-source ops within the componentwise bound of the
  product over the concatenation, and byte for byte what the same op computes launched alone."""
  torch, _lib, lib = env
  case = _case(torch, _lib, lib, B, MS_OPS + SS_OPS, seed=B * 17 + 5)
  n = len(case["ops"])
  order = [8, 0, 1, 9, 2, 3, 4, 10, 5, 6, 7]          # the two kinds interleaved in the op array
  assert sorted(order) == list(range(n))
  group = dict(zip(order, _run(torch, _lib, lib, case, order)))
  fails = []
  for k in range(n):
    fails += _fwd_check(torch, _lib, lib, case, k, group[k])
    alone = _run(torch, _lib, lib, case, [k])[0]
    if not _bytes_equal(group[k], alone):
      fails.append("op %d: grouped output differs from the op launched alone" % k)
  assert not fails, "\n".join(fails)


def test_launches_per_kind(env):
  """One launch per kind per 8 ops: single-source only 1, mixed 2, ten multi-source ops 2."""
  torch, _lib, lib = env
  B = 129
  spec = MS_OPS + SS_OPS + [([70, 70], 64, 1, 1, 1, None), ([5, 60], 40, 1, 0, 0, None)]
  case = _case(torch, _lib, lib, B, spec, seed=7)
  ms, ss = [0, 1, 2, 3, 4, 5, 6, 7, 11, 12], [8, 9, 10]
  for idx, want in ((ss, 1), (ss + ms[:3], 2), (ms, 2)):
    _run(torch, _lib, lib, case, idx)            # descriptors cached
    torch.cuda.synchronize()
    before = _lib.launch_count()
    bufs = _run(torch, _lib, lib, case, idx)
    torch.cuda.synchronize()
    assert _lib.launch_count() - before == want, (idx, want)
    fails = []
    for k, buf in zip(idx, bufs):
      fails += _fwd_check(torch, _lib, lib, case, k, buf)
    assert not fails, "\n".join(fails)


def _bad_variants(_lib, case):
  """(name, mutate(op, keep)) pairs that each make the multi-source op invalid"""
  d = case["ops"][0]
  good = lambda: _lib.FwdSrc(d["xps"][1].data_ptr(), d["wps"][1].data_ptr(), d["widths"][1])

  def with_srcs(srcs, n):
    def f(op, keep):
      arr = (_lib.FwdSrc * max(1, len(srcs)))(*srcs)
      keep.append(arr)
      op.srcs = ctypes.cast(arr, ctypes.POINTER(_lib.FwdSrc))
      op.n_srcs = n
    return f

  def null_srcs(op, keep):
    op.srcs = None
    op.n_srcs = 1

  def bad_piece(**kw):
    s = good()
    for k, v in kw.items():
      setattr(s, k, v)
    return with_srcs([s], 1)

  def own_misaligned(op, keep):      # found while the descriptors are encoded, after the argument checks
    op.xp = d["xps"][0].data_ptr() + 64

  return [("n_srcs < 0", with_srcs([good()], -1)),
          ("n_srcs > 3", with_srcs([good()] * 4, 4)),
          ("srcs NULL", null_srcs),
          ("piece xp NULL", bad_piece(xp=None)),
          ("piece wp NULL", bad_piece(wp=None)),
          ("piece in 0", bad_piece(in_=0)),
          ("piece in < 0", bad_piece(in_=-64)),
          ("piece misaligned", bad_piece(xp=d["xps"][1].data_ptr() + 64)),
          ("own xp misaligned", own_misaligned)]


def test_invalid_pieces_write_nothing(env):
  """A group whose multi-source op is malformed returns ADN_ERR_INVALID, launches nothing, and leaves every output
  of the group, the valid ops' included, as it was: the descriptors of both kinds are encoded before either kind
  is launched."""
  torch, _lib, lib = env
  B = 37
  case = _case(torch, _lib, lib, B, [MS_OPS[0], SS_OPS[0], SS_OPS[1]], seed=11)
  for name, mutate in _bad_variants(_lib, case):
    keep = []
    bufs = [_fwd_buf(torch, _lib, B, d) for d in case["ops"]]
    for b in bufs:
      if b.dim() == 1:
        b.fill_(1.25)                  # sentinel in the plane buffers (the dense ones hold NaN)
    snap = [b.clone() for b in bufs]
    structs = [_struct(_lib, case, d, b, keep) for d, b in zip(case["ops"], bufs)]
    structs = [structs[1], structs[0], structs[2]]
    mutate(structs[1], keep)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    rc = _call(torch, _lib, lib, B, structs)
    torch.cuda.synchronize()
    assert rc == ERR_INVALID, (name, rc)
    assert _lib.launch_count() == before, name
    assert all(_bytes_equal(b, s) for b, s in zip(bufs, snap)), "%s: an output was written" % name


def test_multi_source_in_cuda_graph(env):
  """A mixed group captured in a CUDA graph replays to the bytes of the eager call (no allocation, no sync)."""
  torch, _lib, lib = env
  B = 129
  case = _case(torch, _lib, lib, B, MS_OPS[:4] + SS_OPS[:2], seed=23)
  idx = list(range(len(case["ops"])))
  eager = _run(torch, _lib, lib, case, idx)
  keep = []
  bufs = [_fwd_buf(torch, _lib, B, case["ops"][i]) for i in idx]
  structs = [_struct(_lib, case, case["ops"][i], buf, keep) for i, buf in zip(idx, bufs)]
  arr = (_lib.FwdOp * len(structs))(*structs)
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    _lib.check(lib.adn_dense_fwd_p_group(arr, len(structs), B, _stream(torch)), "captured group")
  for b in bufs:
    b.zero_() if b.dim() == 1 else b.fill_(float("nan"))
  g.replay()
  torch.cuda.synchronize()
  assert all(_bytes_equal(a, b) for a, b in zip(eager, bufs))
