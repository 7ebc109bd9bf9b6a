"""C-ABI surface: the shared library loads on a GPU-less box and exports every
symbol include/dynibar_b200.h declares (no compute calls here)."""

import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dynibar_b200.h")


def _declared():
  src = open(HEADER).read()
  src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
  return sorted(set(re.findall(r"\b(dyn_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
  from dynibar_b200 import _lib
  names = _declared()
  assert len(names) >= 20
  for n in names:
    assert hasattr(_lib.lib, n), "library does not export %s" % n
  # and the ctypes table binds exactly the declared set
  assert sorted(_lib.SIGNATURES) == names


def test_library_is_sm90a_only():
  from dynibar_b200 import _lib
  out = subprocess.run(["cuobjdump", "--list-elf", _lib.LIB_PATH], capture_output=True, text=True)
  if out.returncode != 0:
    return  # cuobjdump not on PATH: nothing to check
  archs = set(re.findall(r"sm_(\d+a?)", out.stdout))
  assert archs == {"90a"}, archs


def test_version_and_error_string_without_gpu():
  from dynibar_b200 import _lib
  assert _lib.lib.dyn_version() >= 100
  # argument validation happens before any CUDA call
  rc = _lib.lib.dyn_sample_rays(None, None, 1.0, 2.0, 4, 8, 0, None, None, None, None, None)
  assert rc == -1 and b"argument check failed" in _lib.lib.dyn_last_error()
  assert _lib.lib.dyn_net_param_count(_lib.NET_DYNAMIC) == 408617
  assert _lib.lib.dyn_net_param_count(_lib.NET_STATIC) == 397905
  assert _lib.lib.dyn_net_param_count(_lib.NET_MOTION) == 533010


def test_containers_match_reference_parameter_counts():
  from dynibar_b200 import synthetic, weights
  model, args = synthetic.make_model(16, 16)
  assert weights.flatten(model.net_coarse_dy).numel() == 408617
  assert weights.flatten(model.net_coarse_st).numel() == 397905
  assert weights.flatten(model.motion_mlp).numel() == 533010


def test_cpu_tensors_are_rejected_loudly():
  import pytest
  import torch
  from dynibar_b200 import render_ray as rr
  with pytest.raises(RuntimeError, match="no CPU fallback"):
    rr.sample_along_camera_ray(torch.zeros(4, 3), torch.ones(4, 3), torch.tensor([[1.0, 2.0]]), 8,
                               det=True)
