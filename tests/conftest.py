import os
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs an H100 (compute capability 9.x)")


# GPU files run leaves-first: the kernel-level parity tests, then the models built from them, then
# the trainers / evaluators / multi-GPU step.  (With `-x` an early failure in a composite test would
# otherwise hide the kernel evidence behind it.)
_GPU_ORDER = ["test_kernels_gpu", "test_attention_gpu", "test_model_gpu", "test_precision_gpu",
              "test_optax_gpu", "test_classifier_gpu", "test_eval_paths", "test_input_pipeline", "test_dist_gpu"]


def _gpu_usable():
  try:
    import torch
    if not torch.cuda.is_available():
      return False
    return torch.cuda.get_device_capability(0)[0] == 9
  except Exception:   # pylint: disable=broad-except
    return False


def pytest_collection_modifyitems(config, items):
  def key(item):
    mod = os.path.splitext(os.path.basename(str(item.fspath)))[0]
    return _GPU_ORDER.index(mod) if mod in _GPU_ORDER else len(_GPU_ORDER)
  items.sort(key=key)     # stable: keeps the in-file order
  if not _gpu_usable():
    skip = pytest.mark.skip(reason="needs a compute-capability 9.x GPU (no CPU fallback exists)")
    for item in items:
      if "gpu" in item.keywords:
        item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built_library():
  """Builds (or re-uses) the in-tree libbv_b200.so; nvcc cross-compiles without a GPU.  On a box
  without the CUDA toolkit the pure-host tests (checkpoints, schedules, oracle) still run; tests that
  load the library then fail on their own with the loader's message."""
  from big_vision_b200 import build
  if shutil.which(build.NVCC) is None and not os.path.exists(build.NVCC):
    return
  build.build(verbose=False)
