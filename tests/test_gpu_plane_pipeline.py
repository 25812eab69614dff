"""The plane GEMM's pipeline (csrc/planes.cu pl_gemm_kernel): consumer warpgroups hand finished tiles to an epilogue
warpgroup through two staging tiles.

* Byte-identical outputs: a fixed, seeded set of forward, dX and dW group launches in both plane formats is hashed
  with SHA-256.  The expected digests were recorded on an H100 80GB HBM3 with the kernel from before the epilogue
  warpgroup, whose consumers ran their own epilogues.  The per-element accumulation order is unchanged, so every
  output byte must be too.
* Shapes aimed at the handoff, each against the float64 componentwise bound of test_gpu_plane_groups.py: many tiles
  per CTA, fewer work items than SMs, 1, 2, 3 and 5 k-blocks per tile, split-K with an odd number of k-blocks per
  split, and consecutive tiles of one CTA from problems with different epilogues.

`python tests/test_gpu_plane_pipeline.py` prints the digests of the current build as JSON.
"""

import hashlib
import json
import os
import sys

import numpy as np
import pytest

if __name__ == "__main__":
  sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.test_gpu_plane_groups import (BWD_OPS, FWD_G11, FWD_WRAP, _bwd_case, _bwd_check, _bwd_run, _fwd_case,
                                         _fwd_check, _fwd_run, _open, _set_format)

pytestmark = pytest.mark.gpu

# forward ops as in test_gpu_plane_groups: (in, out, bias, act, planes out, dropout (seed, layer) or None)
# the first layer of the benchmark's widest candidate at its batch: 256 x 16 = 4096 tiles, ~31 per CTA
FWD_MANY = [(100, 1024, 1, 1, 1, None)]
# 3 + 1 + 2 = 6 work items: far fewer than SMs, one item per CTA
FWD_FEW = [(64, 200, 1, 1, 1, None), (320, 64, 0, 0, 0, None), (192, 65, 1, 0, 1, (71, 0))]
# every problem has the same number of tiles (4 row blocks x 33 column blocks = 132), so the CTAs of a launch walk from
# one problem into the next one tile at a time: consecutive tiles of one CTA differ in K (1, 2, 3, 5 fp16 k-blocks),
# bias, ReLU, dropout and plane versus dense output
FWD_MIXED = [
    (100, 2112, 1, 1, 1, None),
    (64, 2112, 0, 0, 0, None),
    (192, 2112, 1, 1, 1, (72, 1)),
    (320, 2112, 1, 0, 1, None),
    (64, 2112, 1, 1, 0, None),
    (128, 2112, 0, 1, 1, (73, 2)),
]
# backward ops as in test_gpu_plane_groups: (in, out, x_relu_mask, dz_log2_scale, dx_mul (0 = 1), outputs).
# Two one-tile dW problems at batch 28352 = 443 fp16 k-blocks: the split planner (dense_bwd_group) takes its smallest
# split size, ceil(443 / 64) = 7 k-blocks per item, odd, in 64 splits whose last has 2 k-blocks.
BWD_ODD_SPLIT = [(100, 64, 0, 7, 0.0, "dw"), (64, 33, 1, 0, 0.0, "dw")]
BWD_ODD_SPLIT_B = 28352

# (name, kind, spec, batch) of the hashed launches
DIGEST_CASES = [
    ("fwd-g11-b4097", "fwd", FWD_G11, 4097),
    ("fwd-wrap-b128", "fwd", FWD_WRAP, 128),
    ("fwd-mixed-b512", "fwd", FWD_MIXED, 512),
    ("bwd-b256", "bwd", BWD_OPS, 256),
    ("bwd-b8192", "bwd", BWD_OPS, 8192),
    ("bwd-odd-split", "bwd", BWD_ODD_SPLIT, BWD_ODD_SPLIT_B),
]

# recorded on the parent kernel; see the module docstring
EXPECTED = {
    "f16": {
        "bwd-b256": "069f84716c3ee6170cecf14467729d797bd4bfcc30bc947a879dea8c90c6cc59",
        "bwd-b8192": "28c8ccf6f4e0f6af6748ba0b38924ab797ba5323a7be73d1dd8f440caa4d95a6",
        "bwd-odd-split": "bae4a9cf837300b2012f5d4960c57c8dd5b7cdc0013338c887fad2dc6ce0aa5b",
        "fwd-g11-b4097": "ec340caf8d17419f4b32dfe3ece0d86eeddd6bb3adc487f6bb545abd6bb05e7a",
        "fwd-mixed-b512": "8899a890ac6ab39a43b09c558b020ee59b3edf732ec46228b7df362e6e132cf9",
        "fwd-wrap-b128": "2b87250623302880a8a688de29cdaeb349ac75d20a35e7f51d01471b2c2be746",
    },
    "tf32": {
        "bwd-b256": "cf8a31f4fde0caa9fcfd9048ea8a5bc289906144efb6f2f85c3e4ba62cc8382a",
        "bwd-b8192": "2ed37c8970fcd4f67d24d7b95b6965783c68cc0abf364e5f848853f37816adcc",
        "bwd-odd-split": "1ad3ed80afae1c648f955255907ba13a739efdec1a0d3c94094b4e366113f6cd",
        "fwd-g11-b4097": "68d395b54719c9ad39c48b3f263c96b38235fce442a5a9d8b17805b57b6ee236",
        "fwd-mixed-b512": "3121c578b020af0b7e289aa2128444ab115099b7c05092474ed3215596fcc245",
        "fwd-wrap-b128": "c78a2562237a3af1ead11466abecf91a2a42bb8bb77d88b612b798ac620b9268",
    },
}


def _bytes(torch, t):
  torch.cuda.synchronize()
  return t.cpu().numpy().tobytes()


def _case_digest(torch, _lib, lib, kind, spec, B):
  h = hashlib.sha256()
  if kind == "fwd":
    case = _fwd_case(torch, _lib, lib, B, spec, seed=B * 31 + len(spec))
    for buf in _fwd_run(torch, _lib, lib, case, list(range(len(spec)))):
      h.update(_bytes(torch, buf))
  else:
    case = _bwd_case(torch, _lib, lib, B, spec, seed=B + 17)
    for f in _bwd_run(torch, _lib, lib, case, list(range(len(spec)))):
      for key in ("dw", "dxp", "dx", "cs"):
        if f[key] is not None:
          h.update(key.encode())
          h.update(_bytes(torch, f[key]))
  return h.hexdigest()


def digests(formats=("f16", "tf32")):
  """{format: {case: sha256 hex}} of DIGEST_CASES; leaves the plane format as it found it."""
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  out = {}
  try:
    for fmt in formats:
      _set_format(_lib, fmt)
      out[fmt] = {name: _case_digest(torch, _lib, lib, kind, spec, B) for name, kind, spec, B in DIGEST_CASES}
  finally:
    _lib.set_plane_format(before)
  return out


@pytest.fixture(scope="module", params=["f16", "tf32"])
def env(request):
  torch, _lib, lib = _open()
  before = _lib.plane_format()
  _set_format(_lib, request.param)
  _lib.plane_overflow()
  yield request.param, torch, _lib, lib
  _lib.set_plane_format(before)


def test_outputs_byte_identical(env):
  fmt, torch, _lib, lib = env
  got = {name: _case_digest(torch, _lib, lib, kind, spec, B) for name, kind, spec, B in DIGEST_CASES}
  differ = ["%s: %s, want %s" % (n, got[n], EXPECTED[fmt][n]) for n in EXPECTED[fmt] if got[n] != EXPECTED[fmt][n]]
  assert not differ, "\n".join(differ)


FWD_SHAPES = [("many", FWD_MANY, 32768), ("few", FWD_FEW, 256), ("mixed", FWD_MIXED, 512)]


@pytest.mark.parametrize("name,spec,B", FWD_SHAPES, ids=[n for n, _, _ in FWD_SHAPES])
def test_fwd_shapes(env, name, spec, B):
  _, torch, _lib, lib = env
  case = _fwd_case(torch, _lib, lib, B, spec, seed=B * 7 + len(spec))
  bufs = _fwd_run(torch, _lib, lib, case, list(range(len(spec))))
  fails = []
  for k in range(len(spec)):
    fails += _fwd_check(torch, _lib, lib, case, k, bufs[k])
  assert not fails, "\n".join(fails)


def test_dw_odd_split(env):
  _, torch, _lib, lib = env
  case = _bwd_case(torch, _lib, lib, BWD_ODD_SPLIT_B, BWD_ODD_SPLIT, seed=3)
  bufs = _bwd_run(torch, _lib, lib, case, list(range(len(BWD_ODD_SPLIT))))
  fails = []
  for k in range(len(BWD_ODD_SPLIT)):
    fails += _bwd_check(torch, _lib, lib, case, k, bufs[k])
  assert not fails, "\n".join(fails)


if __name__ == "__main__":
  print(json.dumps(digests(), indent=1, sort_keys=True))
