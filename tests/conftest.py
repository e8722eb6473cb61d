import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
  if p not in sys.path:
    sys.path.insert(0, p)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
  import torch
  if torch.cuda.is_available():
    return
  skip = pytest.mark.skip(reason="no CUDA device")
  for item in items:
    if "gpu" in item.keywords:
      item.add_marker(skip)
