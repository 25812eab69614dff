import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
  try:
    import torch
    has_gpu = torch.cuda.is_available()
  except Exception:   # pragma: no cover
    has_gpu = False
  if has_gpu:
    return
  skip = pytest.mark.skip(reason="no CUDA device in this container")
  for item in items:
    if "gpu" in item.keywords:
      item.add_marker(skip)


@pytest.fixture(scope="session")
def built_lib():
  """The in-tree CUDA extension; built on demand (nvcc cross-compiles without a GPU)."""
  import __graft_entry__ as g
  g.build()
  from adanet_b200 import _lib
  return _lib.load()


@pytest.fixture(autouse=True)
def _default_plane_format(request):
  """A GPU test that triggers the fp16 -> TF32 plane fallback (sticky per process, core/search.py) must not change
  the format the following tests run on."""
  if "gpu" not in request.keywords:
    yield
    return
  from adanet_b200 import _lib
  try:
    before = _lib.plane_format()
  except Exception:
    yield
    return
  yield
  if _lib.plane_format() != before:
    _lib.set_plane_format(before)
    _lib.plane_overflow()
