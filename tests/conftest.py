import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
  if p not in sys.path:
    sys.path.insert(0, p)


def pytest_configure(config):
  config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
  if torch.cuda.is_available():
    return
  skip = pytest.mark.skip(reason="no CUDA device")
  for item in items:
    if "gpu" in item.keywords:
      item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
  def load(name):
    return torch.load(os.path.join(ROOT, "tests", "golden", name + ".pt"),
                      weights_only=False)
  return load
